"""The LDE as coefficients plus one coset (p3gpu_lde_coefficients_dev, p3gpu_lde_coset_block_dev) against the whole LDE.

For both fields, added_bits 1 to 3 and shapes on each forward path the coset DFT takes — the TMA pass pipeline (width a multiple of
4, 8 to 8192 columns, passes of fewer than 10 layers), the cp.async tile kernel (10-layer passes, a width above 8192), the generic
kernel (a width that is not a multiple of 4, small heights), the band kernel as the last pass (narrow widths at 2^14 and 2^20 rows)
and the one-row constant — every coset written over a poisoned buffer must equal its row range of p3gpu_coset_lde_batch_dev, word for
word.  The conversion to coefficients runs in the trace's own storage: the device's free memory does not drop by a trace."""
import numpy as np
import pytest
import torch

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import Gpu

pytestmark = pytest.mark.gpu
POISON = -1                     # 0xFFFFFFFF: not a canonical word of either field

SHAPES = [(0, 5), (4, 12), (7, 3), (10, 7), (12, 100), (14, 16), (14, 64), (16, 8200), (18, 36), (20, 100)]
CASES = [(f, ab, log_h, w) for f in (BabyBear, KoalaBear) for ab in (1, 2, 3) for log_h, w in SHAPES]


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return Gpu(0)


def _random(f, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, f.P, (h, w), dtype=torch.int32, device="cuda", generator=g)


@pytest.mark.parametrize("f,added_bits,log_h,w", CASES, ids=[f"{f.name}-b{ab}-2^{lh}x{w}" for f, ab, lh, w in CASES])
def test_every_coset_equals_its_rows_of_the_lde(gpu, f, added_bits, log_h, w):
    h = 1 << log_h
    trace = _random(f, h, w, 1000 * log_h + w + added_bits)
    shift = f.generator if (log_h + added_bits) % 2 else f.to_monty(7)        # the PCS's shift and another one
    lde = gpu.coset_lde_batch(f.id, trace, added_bits, shift, bitrev_rows=True)
    coeffs = gpu.lde_coefficients(f.id, trace.clone())
    out = torch.full((h, w), POISON, dtype=torch.int32, device="cuda")
    for k in range(1 << added_bits):
        out.fill_(POISON)
        gpu.lde_coset_block(f.id, coeffs, added_bits, shift, k, out=out)
        want = lde[k * h:(k + 1) * h]
        if not torch.equal(out, want):
            bad = (out != want).nonzero()
            r, c = int(bad[0, 0]), int(bad[0, 1])
            pytest.fail(f"coset {k}: {bad.shape[0]} words differ, first at row {r} column {c}: "
                        f"{int(out[r, c]) & 0xFFFFFFFF:#x} against {int(want[r, c]) & 0xFFFFFFFF:#x}")


def test_the_coefficients_are_computed_in_place():
    f, h, w = KoalaBear, 1 << 20, 256                             # a 1 GiB trace
    g = Gpu(0)                                                   # a fresh context: nothing cached yet
    trace = _random(f, h, w, 7)
    keep = trace.clone()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    torch.cuda.reset_peak_memory_stats()
    alloc0 = torch.cuda.memory_allocated()
    ptr = trace.data_ptr()
    coeffs = g.lde_coefficients(f.id, trace)
    torch.cuda.synchronize()
    assert coeffs.data_ptr() == ptr
    assert torch.cuda.max_memory_allocated() == alloc0
    drop = free0 - torch.cuda.mem_get_info()[0]
    assert drop < h * w * 4 // 4, f"free memory dropped by {drop} bytes converting a {h * w * 4}-byte trace"
    # and the coefficients are the LDE's: coset 1 of blowup 2 against the whole LDE of the kept copy
    lde = g.coset_lde_batch(f.id, keep, 1, f.generator, bitrev_rows=True)
    assert torch.equal(g.lde_coset_block(f.id, coeffs, 1, f.generator, 1), lde[h:])
    g.close()


def test_bad_arguments_are_refused(gpu):
    f = KoalaBear
    coeffs = _random(f, 16, 8, 3)
    with pytest.raises(_lib.P3GpuError, match="coset 4 of an LDE with 4 cosets"):
        gpu.lde_coset_block(f.id, coeffs, 2, f.generator, 4)
    with pytest.raises(_lib.P3GpuError, match="cannot overwrite the coefficients"):
        gpu.lde_coset_block(f.id, coeffs, 1, f.generator, 0, out=coeffs)
    with pytest.raises(_lib.P3GpuError, match="not a power of two"):
        gpu.lde_coefficients(f.id, _random(f, 12, 8, 4))
