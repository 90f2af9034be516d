"""The coset LDE's tile-major plan (csrc/ntt.cu: make_tile_major_tensor_maps, ntt_band_pass_kernel<F, R, 8, true, false>).

When the 8-CTA band pass takes the LDE's last pass (more than 48 columns, an eighth of a band within a ring slot), the fused middle
pass's column tile divides the width and there are at least two tiles, the fused pass stores each finished tile as one dense block
of its own scratch, and the band pass gathers each part's rows from those blocks with one tensor copy.  Every other shape keeps the
dense layout, and so do P3GPU_NTT_GATHER=0 and P3GPU_NTT_BAND=0.  At 2^14 rows each case is checked against the CPU oracle; at 2^18
and 2^20 rows the result must be bit-identical to the dense layout on the band pass and on the tile kernel, written over poisoned,
guarded outputs after a dirty call."""
import numpy as np
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_gpu_lde_band import _lde_poisoned
from test_gpu_lde_first_band import _strided_first
from test_gpu_lde_paths import G, POISON, _lde_mid_tile_width, run_lde_checked

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]
BAND_NARROW_W = 48          # csrc/ntt.cu: up to 48 columns the last pass runs on the 4-CTA kernel, which has no gather mode
BAND_SLOT_BYTES = 50 * 1024
GATHER_NAME = "true, false>"   # the gather instance's template arguments (GATHER, STRIDED)


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def _gathers(log_h, w):
    """Whether coset_lde_impl takes the tile-major plan for a three-launch LDE of 2^log_h x w."""
    r, ct = log_h // 2, _lde_mid_tile_width(w)
    band = w % 4 == 0 and ((w * 4) << r) // 8 <= BAND_SLOT_BYTES
    return band and w > BAND_NARROW_W and ct != 0 and w % ct == 0 and w // ct >= 2


# 64 / 60 / 100: 16- and 20-column tiles; 72: the runtime-width instance (12-column tiles); 52: a ragged last tile (20 + 20 + 12);
# 48: the narrow band kernel
SMALL_WIDTHS = [64, 60, 100, 72, 52, 48]


def test_small_widths_cover_both_plans():
    assert [_gathers(14, w) for w in SMALL_WIDTHS] == [True, True, True, True, False, False]


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", SMALL_WIDTHS)
@pytest.mark.parametrize("added_bits", [0, 1, 2])
def test_gather_small_matches_oracle(gpu, f, w, added_bits, monkeypatch):
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^14 rows take the TMA pipeline by default; the three-launch path needs it off
    m = O.random_matrix(f.id, 1 << 14, w, seed=9900 + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)


def _check_body(what, out, f):
    u = out.cpu().numpy().view(np.uint32)
    assert (u[:G] == POISON).all() and (u[-G:] == POISON).all(), f"{what}: wrote outside its output"
    body = u[G:-G]
    assert (body < f.P).all(), f"{what}: {int((body >= f.P).sum())} words not canonical (never written?)"


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w,added_bits", [(18, 200, 1), (18, 96, 2), (20, 64, 1), (20, 100, 0), (20, 100, 1), (20, 100, 2)])
def test_gather_matches_dense_layout(gpu, f, log_h, w, added_bits, monkeypatch):
    assert _gathers(log_h, w)
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    h = 1 << log_h
    gen = torch.Generator(device="cuda").manual_seed(77 * log_h + w + 1000 * added_bits)
    x = torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen)
    what = f"{f.name} LDE 2^{log_h} x {w}, added_bits {added_bits}"
    got = _lde_poisoned(gpu, f, x, h, w, added_bits)
    _check_body(what, got, f)
    for env in ("P3GPU_NTT_GATHER", "P3GPU_NTT_BAND"):
        monkeypatch.setenv(env, "0")
        want = _lde_poisoned(gpu, f, x, h, w, added_bits)
        monkeypatch.delenv(env)
        bad = got != want
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0]) - G
            pytest.fail(f"{what}: {int(bad.sum())} words differ from the dense layout with {env}=0; first at row {i // w}, column {i % w}")


def _last_call_kernels(gpu, f, log_h, w, added_bits=1, calls=4):
    """The kernel names of one p3gpu_coset_lde_batch_dev call (three launches), in launch order, from torch.profiler.  The profiler
    can lose kernels that start soon after it begins recording, even behind a spin kernel, so one profile holds `calls` identical
    calls and the last call's three launches are taken, once the two calls before it were recorded with the same three names."""
    h = 1 << log_h
    x = torch.zeros((h * w,), dtype=torch.int32, device="cuda")
    out = torch.empty(((h << added_bits) * w,), dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    call = lambda: _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, out.data_ptr(), 1))
    call()   # the first call of a shape may also build its twiddle heaps
    n0 = gpu.launches
    call()
    torch.cuda.synchronize()
    assert gpu.launches - n0 == 3, f"LDE 2^{log_h} x {w}: {gpu.launches - n0} launches: the case left the three-launch path"
    for _ in range(5):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1 << 24)
            for _ in range(calls):
                call()
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
        names = [e.name for e in events if "spin_kernel" not in e.name]
        if len(names) >= 9 and names[-3:] == names[-6:-3] == names[-9:-6]:
            return names[-3:]
    pytest.fail(f"torch.profiler did not record two whole calls of {calls}: {names}")


@pytest.mark.parametrize("log_h,w", [(20, 100), (20, 64), (20, 48), (20, 104), (18, 200), (14, 800), (14, 72), (14, 52)])
def test_gather_dispatch(gpu, log_h, w, monkeypatch):
    # 104 columns at 2^20 rows make an eighth of a band larger than a ring slot; 52 has a ragged column tile.  (P3GPU_NTT_BAND=0
    # leaves no band kernel at all: test_gpu_lde_band checks that.)
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    names = _last_call_kernels(gpu, KoalaBear, log_h, w)
    assert (GATHER_NAME in names[2] and "ntt_band_pass_kernel" in names[2]) == _gathers(log_h, w), names
    assert not any(GATHER_NAME in n for n in names[:2]), names
    if w in (100, 200):
        assert _strided_first(names), names
    monkeypatch.setenv("P3GPU_NTT_GATHER", "0")
    names = _last_call_kernels(gpu, KoalaBear, log_h, w)
    assert not any(GATHER_NAME in n for n in names), names


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_gather_back_to_back(gpu, f, monkeypatch):
    # ten LDEs on one stream with no synchronisation, then a wider blow-up that regrows the tile-major scratch between calls
    calls = [(100, 1)] * 10 + [(96, 2)]
    h = 1 << 20
    gpu._use_torch_stream()
    gen = torch.Generator(device="cuda").manual_seed(6161 + f.id)
    xs, outs = [], []
    for w, added_bits in calls:
        xs.append(torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen))
        outs.append(torch.full(((h << added_bits) * w,), -1, dtype=torch.int32, device="cuda"))
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, xs[-1].data_ptr(), h, w, added_bits, f.generator, outs[-1].data_ptr(), 1))
    torch.cuda.synchronize()
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    for i, ((w, added_bits), x, out) in enumerate(zip(calls, xs, outs)):
        want = torch.empty_like(out)
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, want.data_ptr(), 1))
        torch.cuda.synchronize()
        bad = out != want
        if bool(bad.any()):
            j = int(torch.nonzero(bad)[0])
            pytest.fail(f"{f.name} LDE 2^20 x {w}, added_bits {added_bits}, call {i} of {len(calls)}: {int(bad.sum())} words differ "
                        f"from the tile kernel; first at row {j // w}, column {j % w}")
