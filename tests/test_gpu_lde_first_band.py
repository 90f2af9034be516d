"""Inverse pass 1 of the three-launch coset LDE on strided units (csrc/ntt.cu: ntt_band_pass_kernel<F, R, 8, true>).

The first pass applies inverse layers 0 .. r-1 to the unit of rows L + 2^r * i, i < 2^r (2^2r rows).  It runs on the band pass's
8-CTA clusters, each CTA's eighth of a unit moved by one 3-D tensor copy in and one out, when an eighth (2^r / 8 rows x w words)
fits a 50 KB ring slot, w % 4 == 0, BAND_FIRST_MIN_W <= w <= 256, and the buffers are 16-byte aligned.  Every other shape keeps the
tile kernel (ntt_pass_fast_kernel), and P3GPU_NTT_BAND=0 forces it.  Each case writes into a poisoned, guarded output after a
dirty call, and must be bit-identical to the tile kernel; at 2^14 rows it is also checked against the CPU oracle, and at 2^18 and
2^20 rows _band_against_tile_kernel checks the tile kernel's result against tests/ntt_reference.py on the device."""
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_gpu_lde_band import _band_against_tile_kernel
from test_gpu_lde_paths import run_lde_checked

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]
BAND_FIRST_MIN_W = 100  # csrc/ntt.cu: narrower matrices keep the tile kernel for the first pass


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def _kernels_launched(gpu, f, log_h, w, added_bits=1):
    """The kernel names one p3gpu_coset_lde_batch_dev call launches, in launch order (torch.profiler).  The profiler can lose
    the kernel that starts right after it begins recording: a spin kernel (torch.cuda._sleep, left out) goes first, and the
    profile is taken again while it holds fewer kernels than the library counted.  A profile that still misses some fails here,
    so that a check that no band kernel ran cannot pass on an incomplete list."""
    h = 1 << log_h
    x = torch.zeros((h * w,), dtype=torch.int32, device="cuda")
    out = torch.empty(((h << added_bits) * w,), dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    call = lambda: _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, out.data_ptr(), 1))
    call()
    torch.cuda.synchronize()
    for _ in range(3):
        n0 = gpu.launches
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1 << 24)
            call()
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
        names = [e.name for e in events if "spin_kernel" not in e.name]
        n = gpu.launches - n0
        if len(names) == n:
            return names
    pytest.fail(f"torch.profiler recorded {len(names)} of the {n} kernels the library launched: {names}")


def _strided_first(names):
    return len(names) == 3 and "ntt_band_pass_kernel" in names[0] and "true>" in names[0]


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [4, 8, 96, 100, 256])
@pytest.mark.parametrize("added_bits", [1, 2])
def test_first_band_small_matches_oracle(gpu, f, w, added_bits, monkeypatch):
    # 2^14 rows (7 + 7 layers): a 16-row eighth; 4, 8 and 96 columns are below BAND_FIRST_MIN_W and check the tile kernel beside it
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^14 rows take the TMA pipeline by default; the three-launch path needs it off
    m = O.random_matrix(f.id, 1 << 14, w, seed=8800 + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)
    _band_against_tile_kernel(gpu, f, 14, w, added_bits, monkeypatch)


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w,added_bits", [(18, 96, 1), (18, 200, 1), (20, 4, 1), (20, 64, 1), (20, 100, 1), (20, 100, 2),
                                                (20, 104, 1)])
def test_first_band_matches_tile_kernel(gpu, f, log_h, w, added_bits, monkeypatch):
    # 2^20 x 104: an eighth of 53,248 bytes does not fit the ring slot, so both passes fall back to the tile kernel
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    _band_against_tile_kernel(gpu, f, log_h, w, added_bits, monkeypatch)


@pytest.mark.parametrize("log_h,w,strided", [(20, 100, True), (18, 200, True), (20, 104, False), (14, 800, False),
                                             (20, BAND_FIRST_MIN_W - 4, False), (20, BAND_FIRST_MIN_W, True)])
def test_first_band_dispatch(gpu, log_h, w, strided, monkeypatch):
    # 800 columns exceed the 256-element tensor box; 104 at 2^20 rows make an eighth larger than a ring slot
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    names = _kernels_launched(gpu, KoalaBear, log_h, w)
    assert len(names) == 3, names
    assert _strided_first(names) == strided, names
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    names = _kernels_launched(gpu, KoalaBear, log_h, w)
    assert not any("ntt_band_pass" in n for n in names), names


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_first_band_back_to_back(gpu, f, monkeypatch):
    # ten LDEs on one stream with no synchronisation: each runs the strided pass and then, after the fused launch, the band pass
    # of the same kernel template, so ring, mbarrier or store state leaking from one launch into the next shows as a mismatch
    h, w, H = 1 << 20, 100, 1 << 21
    gpu._use_torch_stream()
    gen = torch.Generator(device="cuda").manual_seed(5151 + f.id)
    xs, outs = [], []
    for _ in range(10):
        xs.append(torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen))
        outs.append(torch.full((H * w,), -1, dtype=torch.int32, device="cuda"))
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, xs[-1].data_ptr(), h, w, 1, f.generator, outs[-1].data_ptr(), 1))
    torch.cuda.synchronize()
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    want = torch.empty((H * w,), dtype=torch.int32, device="cuda")
    for i, (x, out) in enumerate(zip(xs, outs)):
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, 1, f.generator, want.data_ptr(), 1))
        torch.cuda.synchronize()
        bad = out != want
        if bool(bad.any()):
            j = int(torch.nonzero(bad)[0])
            pytest.fail(f"{f.name} LDE 2^20 x {w}, call {i} of 10: {int(bad.sum())} words differ from the tile kernel; first at row "
                        f"{j // w}, column {j % w}")
