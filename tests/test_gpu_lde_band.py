"""Forward pass 2 of the three-launch coset LDE on whole-row bands (csrc/ntt.cu: ntt_band_pass_kernel, 8-CTA clusters; up to
48 columns ntt_band_pass_narrow_kernel, 4-CTA clusters).

The band pass takes the LDE's last pass when an eighth of a band (2^r / 8 rows x w columns, r = log_h / 2) fits its 50 KB ring
slot (BAND_CL, BAND_SLOT_BYTES) and the width is a multiple of 4: w <= 800 at 2^14 rows, <= 200 at 2^18, <= 100 at 2^20.  Every
other width keeps the tile kernel (ntt_pass_fast_kernel), and P3GPU_NTT_BAND=0 forces it.  Each case writes into a poisoned, guarded output and must be
bit-identical to the same call on the tile kernel; at 2^14 rows it is also checked against the CPU oracle, and at 2^18 and 2^20 the
tile kernel's result is checked against tests/ntt_reference.py on the device."""
import numpy as np
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
import ntt_reference as R
from test_gpu_lde_paths import G, POISON, check_matrix, run_lde_checked

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def _lde_poisoned(gpu, f, x, h, w, added_bits):
    """The LDE of the device matrix x into a fresh buffer of 0xFFFFFFFF words with G guard words on each side, after a dirty
    call on other data (so that no scratch or output block holds this input's result from an earlier call); asserts that the
    call takes the three-launch path."""
    H = h << added_bits
    gen = torch.Generator(device="cuda").manual_seed(h * w + added_bits + 7)
    dirty = torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen)
    out = torch.full((H * w + 2 * G,), -1, dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, dirty.data_ptr(), h, w, added_bits, f.generator, out.data_ptr() + 4 * G, 1))
    out.fill_(-1)
    n0 = gpu.launches
    _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, out.data_ptr() + 4 * G, 1))
    assert gpu.launches - n0 == 3, f"LDE 2^{h.bit_length() - 1} x {w}: {gpu.launches - n0} launches: the case left the three-launch path"
    torch.cuda.synchronize()
    return out


def _band_against_tile_kernel(gpu, f, log_h, w, added_bits, monkeypatch):
    h = 1 << log_h
    gen = torch.Generator(device="cuda").manual_seed(31 * log_h + w + 1000 * added_bits)
    x = torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen)
    band = _lde_poisoned(gpu, f, x, h, w, added_bits)
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    tile = _lde_poisoned(gpu, f, x, h, w, added_bits)
    monkeypatch.delenv("P3GPU_NTT_BAND")
    what = f"{f.name} LDE 2^{log_h} x {w}, added_bits {added_bits}"
    u = band.cpu().numpy().view(np.uint32)
    assert (u[:G] == POISON).all() and (u[-G:] == POISON).all(), f"{what}: band pass wrote outside its output"
    body = u[G:-G]
    assert (body < f.P).all(), f"{what}: {int((body >= f.P).sum())} words not canonical (never written?)"
    if log_h >= 18:   # too large for the CPU oracle: the tile kernel's result against the reference transform on the device
        H, xm = h << added_bits, x.view(h, w)
        check_matrix(f, tile[G:G + H * w].view(H, w), lambda c0, c1: R.coset_lde(f, xm[:, c0:c1], added_bits, f.generator),
                     lambda row, col: f"coset block {row >> log_h}", f"{what} on the tile kernel")
    bad = band != tile
    if bool(bad.any()):
        i = int(torch.nonzero(bad)[0]) - G
        pytest.fail(f"{what}: {int(bad.sum())} words differ from the tile kernel; first at row {i // w}, column {i % w}")


def _band_kernel_launched(gpu, f, log_h, w):
    """Whether p3gpu_coset_lde_batch_dev launches ntt_band_pass_kernel for this shape (torch.profiler kernel names)."""
    h = 1 << log_h
    x = torch.zeros((h * w,), dtype=torch.int32, device="cuda")
    out = torch.empty(((2 * h) * w,), dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, 1, f.generator, out.data_ptr(), 1))
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, 1, f.generator, out.data_ptr(), 1))
        torch.cuda.synchronize()
    return any("ntt_band_pass_kernel" in e.key for e in prof.key_averages())


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [4, 8, 96, 100, 800])
@pytest.mark.parametrize("added_bits", [1, 2])
def test_band_pass_small_matches_oracle(gpu, f, w, added_bits, monkeypatch):
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^14 rows take the TMA pipeline by default; the three-launch path needs it off
    m = O.random_matrix(f.id, 1 << 14, w, seed=7700 + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)
    _band_against_tile_kernel(gpu, f, 14, w, added_bits, monkeypatch)


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w", [(18, 4), (18, 8), (18, 96), (18, 100), (18, 200), (20, 4), (20, 8), (20, 96), (20, 100), (20, 104)])
def test_band_pass_matches_tile_kernel(gpu, f, log_h, w, monkeypatch):
    # 2^20 x 104: an eighth of a band, 52 KB, does not fit the ring slot, so both calls run the tile kernel (the fallback)
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    _band_against_tile_kernel(gpu, f, log_h, w, 1, monkeypatch)


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_band_pass_four_cosets_full_height(gpu, f, monkeypatch):
    _band_against_tile_kernel(gpu, f, 20, 100, 2, monkeypatch)


@pytest.mark.parametrize("log_h,w,band", [(20, 100, True), (20, 104, False), (18, 200, True), (18, 204, False), (14, 800, True)])
def test_band_pass_dispatch(gpu, log_h, w, band, monkeypatch):
    # 104 columns at 2^20 rows (204 at 2^18) make an eighth of a band of 52 KB (51 KB), more than a ring slot: the tile kernel runs
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    assert _band_kernel_launched(gpu, KoalaBear, log_h, w) == band
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    assert not _band_kernel_launched(gpu, KoalaBear, log_h, w)

