"""Coset LDEs and DFTs at shapes no other test runs, every word checked on the device against tests/ntt_reference.py.

Each case goes through run_lde_checked / run_dft_checked (test_gpu_lde_paths) with a DeviceInput: a dirty call on other data
first, then the call into a poisoned output with guard words on both sides, and every word must be canonical and equal to the
reference.  Each case also pins the number of kernels it launches, which identifies its path (pass plan, column chunks, one
network per coset), so that a dispatch change fails here instead of silently moving the case off the path it checks:
  * the top of the two-adic subgroup: KoalaBear 2^23 -> 2^24, BabyBear 2^26 -> 2^27 and 2^24 -> 2^27, and the DFT kinds at
    2^24 (KoalaBear) and 2^27 (BabyBear);
  * both sides of lde_tiled_impl's scratch limit: the tiled pipeline gives up when the forward intermediate of one column chunk
    (2^added_bits * h * chunk words, chunk >= min(64, width rounded up to 8)) would exceed 8 GiB, and the LDE runs as plain
    networks on dense buffers instead (both cases are wide enough that the tiled pipeline would run two column chunks, so the
    launch count tells the two paths apart);
  * more than 2^31 input words and 2^32 output words (2^20 x 2056, blowup 2, both fields) on the fused three-launch path and on the
    tiled pipeline (P3GPU_NTT_PIPE=1), where 32-bit index arithmetic would wrap;
  * natural-order rows above 2^20, the DFT kinds above 2^20 at a wide and a narrow width, and the host-pointer entry point at the
    2^20 x 100 shape bench.py's e2e leg runs.

Every case runs on a context of its own: the library's scratch buffers are cudaMalloc'd outside torch's allocator and only grow,
so they are freed with the context after each case.  The peak device memory of each case (torch's peak plus what the context
held) is recorded as the test property peak_device_gb (pytest --junitxml)."""
import pytest
import torch

import ntt_reference as R
from test_gpu_lde_paths import G, DeviceInput, _check_output, run_dft_checked, run_lde_checked

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import Gpu

pytestmark = pytest.mark.gpu
BB, KB = BabyBear, KoalaBear
KINDS = {"DFT": _lib.DFT, "iDFT": _lib.IDFT, "coset_DFT": _lib.COSET_DFT, "coset_iDFT": _lib.COSET_IDFT}


def _used():
    free, total = torch.cuda.mem_get_info()
    return total - free


@pytest.fixture
def gpu(record_property):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    used0, reserved0 = _used(), torch.cuda.memory_reserved()
    g = Gpu(0)
    yield g
    torch.cuda.synchronize()
    held = (_used() - used0) - (torch.cuda.memory_reserved() - reserved0)   # the context's scratch, twiddle heaps and buffers
    g.close()
    torch.cuda.empty_cache()
    record_property("peak_device_gb", round((torch.cuda.max_memory_reserved() + held) / 1e9, 1))


def _needs(gb):
    free = torch.cuda.mem_get_info()[0]
    if free < gb * 1e9:
        pytest.fail(f"needs {gb} GB, {free / 1e9:.1f} GB free")


# ------------------------------------------------------------------------------------------ top of the two-adic subgroup
@pytest.mark.parametrize("f,log_h,w,added_bits,launches", [
    (KB, 23, 4, 1, 6),        # no 16-byte rows: inverse and forward network on the cp.async kernel, 8 + 8 + 7 layers
    (KB, 23, 100, 1, 12),     # the tiled pipeline in two column chunks (64 + 36), six launches each
    # the tiled pipeline in one column chunk (9 + 9 + 8 layers): the widest one the scratch limit allows here (2 cosets x 2^26
    # rows x 16 columns = 8 GiB), so the launch count cannot tell it from the dense networks it would otherwise fall back to
    (BB, 26, 8, 1, 6),
    (BB, 24, 4, 3, 6),        # the cp.async kernel, all 8 cosets in each forward launch
    (BB, 24, 8, 3, 6),        # the tiled pipeline in one chunk (as at 2^26, at most 16 columns fit the limit): count as above
], ids=lambda v: v.name if hasattr(v, "name") else None)
def test_lde_to_the_top_of_two_adicity(gpu, f, log_h, w, added_bits, launches):
    assert log_h + added_bits == f.TWO_ADICITY
    run_lde_checked(gpu, f, DeviceInput(1 << log_h, w, seed=log_h * 1000 + w), added_bits, f.generator, launches=launches)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f,log_h,w", [(KB, 24, 4), (BB, 27, 8)], ids=lambda v: v.name if hasattr(v, "name") else None)
def test_dft_kinds_at_the_top_of_two_adicity(gpu, kind, f, log_h, w):
    # three passes (8 + 8 + 8 layers on the cp.async kernel at 4 columns, 9 + 9 + 9 on the pipeline at 8); the coset iDFT adds
    # its row scaling
    assert log_h == f.TWO_ADICITY
    k = KINDS[kind]
    run_dft_checked(gpu, f, k, DeviceInput(1 << log_h, w, seed=k + 10 * w), f.to_monty(0x2345678 + log_h),
                    launches=4 if k == _lib.COSET_IDFT else 3)


# ------------------------------------------------------------------------------------------ the tiled pipeline's scratch limit
@pytest.mark.parametrize("log_h,w,launches", [
    (22, 100, 12),   # 8 cosets x 2^22 rows x 64-column chunks x 4 bytes = 8 GiB exactly: the tiled pipeline, chunks of 64 + 36
    # 8 cosets x 2^23 rows x 64-column chunks x 4 bytes = 16 GiB: one inverse and one forward network on dense buffers; the tiled
    # pipeline would take 12 launches here (chunks of 64 + 8), so the count tells the two apart
    (23, 72, 6),
])
def test_lde_on_both_sides_of_the_tiled_scratch_limit(gpu, log_h, w, launches):
    run_lde_checked(gpu, BB, DeviceInput(1 << log_h, w, seed=log_h + w), 3, BB.generator, launches=launches)


# ------------------------------------------------------------------------------------------ past 2^31 / 2^32 words
@pytest.mark.parametrize("f", [BB, KB], ids=lambda f: f.name)
@pytest.mark.parametrize("pipe_mode,launches", [
    (None, 3),       # 2056 columns: the three-launch path with 20-column tiles, 103 of them (the last one 16 wide)
    ("1", 4 * 17),   # the tiled pipeline in 128-column chunks: 16 of them and one of 8 columns, four launches each
], ids=["fused", "tiled"])
def test_lde_past_2_32_output_words(gpu, f, pipe_mode, launches, monkeypatch):
    h, w = 1 << 20, 2056
    assert h * w > 1 << 31 and 2 * h * w > 1 << 32
    # input 8.6 GB, output 17.2 GB, the fused path's coefficient scratch 8.6 GB, the reference's column chunk about 5 GB
    _needs(42)
    if pipe_mode:
        monkeypatch.setenv("P3GPU_NTT_PIPE", pipe_mode)
    run_lde_checked(gpu, f, DeviceInput(h, w, seed=2056), 1, f.generator, launches=launches)


# ------------------------------------------------------------------------------------------ natural-order rows
@pytest.mark.parametrize("added_bits", [1, 2])
@pytest.mark.parametrize("f", [BB, KB], ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w", [(21, 100), (22, 8)])
def test_natural_order_rows_above_2_20(gpu, f, log_h, w, added_bits):
    # the inverse network, then one forward network per coset, whose last pass writes network position i of coset c to row
    # (bitrev(i) << added_bits) + c: three passes each
    run_lde_checked(gpu, f, DeviceInput(1 << log_h, w, seed=log_h + w + added_bits), added_bits, f.generator, bitrev_rows=False,
                    launches=3 + 3 * (1 << added_bits))


# ------------------------------------------------------------------------------------------ DFT kinds above 2^20
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f", [BB, KB], ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w", [(22, 300), (21, 4)])
def test_dft_kinds_above_2_20(gpu, kind, f, log_h, w):
    # three passes (the pipeline at 300 columns, the cp.async kernel at 4); the coset iDFT adds its row scaling
    k = KINDS[kind]
    run_dft_checked(gpu, f, k, DeviceInput(1 << log_h, w, seed=k + log_h), f.to_monty(0x1234567 + w),
                    launches=4 if k == _lib.COSET_IDFT else 3)


# ------------------------------------------------------------------------------------------ host pointers
@pytest.mark.parametrize("chunks,launches", [
    (None, 3),       # one chunk: the three-launch path on the whole matrix
    ("3", 3 * 3),    # column chunks of 36, 32 and 32, three launches each
], ids=["one_chunk", "three_chunks"])
def test_host_pointer_lde_at_the_e2e_shape(gpu, chunks, launches, monkeypatch):
    # p3gpu_coset_lde_batch with pinned host buffers at bench.py's e2e shape (KoalaBear 2^20 x 100, blowup 2), by default in one
    # chunk and with P3GPU_E2E_CHUNKS=3 as a pipeline of column chunks on three streams
    if chunks:
        monkeypatch.setenv("P3GPU_E2E_CHUNKS", chunks)
    f, h, w = KB, 1 << 20, 100
    H = 2 * h
    x = torch.empty(h * w, dtype=torch.int32).pin_memory()
    out = torch.empty(H * w + 2 * G, dtype=torch.int32).pin_memory()
    call = lambda: _lib.check(gpu.L.p3gpu_coset_lde_batch(gpu.h, f.id, x.data_ptr(), h, w, 1, f.generator, out.data_ptr() + 4 * G, 1))
    x.random_(0, f.P, generator=torch.Generator().manual_seed(1))
    call()                                                                   # dirty call on other data
    xd = torch.randint(0, f.P, (h, w), dtype=torch.int32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100))
    x.copy_(xd.view(-1))
    out.fill_(-1)
    n0 = gpu.launches
    call()
    what = f"{f.name} host-pointer LDE 2^20 x {w}, P3GPU_E2E_CHUNKS={chunks}"
    assert gpu.launches - n0 == launches, f"{what}: {gpu.launches - n0} launches instead of {launches}: the case left the path it pins"
    _check_output(f, out.cuda(), 0, H, w, lambda c0, c1: R.coset_lde(f, xd[:, c0:c1], 1, f.generator), lambda r, c: f"coset {r >> 20}",
                  what)
