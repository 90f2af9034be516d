"""Edge cases of the producer-warp ring of the three-launch coset LDE (csrc/ntt.cu: ntt_pass_fast_kernel and
ntt_lde_mid_kernel, PROD).  A CTA runs one producer warp and walks its tiles through two buffers: the producer loads tile k + 2
into buffer k % 2 only after the consumers and the tile's tensor-copy store(s) have left it, and the fused kernel's consumers
wait for each coset's store to be read out before the next coset rewrites the buffer.  The cases below change how many tiles
each persistent CTA of the pass kernel gets (one CTA per SM: 132 on an H100 SXM; at 2^14 rows the fused kernel's small tiles
fit several CTAs per SM, which then take one tile each):
  * 2^14 rows (7 + 7 layers), width 4: 128 tiles per launch, fewer than the SMs, so every CTA has exactly one tile and the
    forward pass with two cosets gives CTAs one or two;
  * 2^14 x 40 (two 20-column tiles): 256 tiles, two per CTA on most SMs (an even count);
  * 2^14 x 60 (three 20-column tiles): 384 tiles, three per CTA on most SMs (an odd count);
  * 2^20 x 100 and 2^20 x 16: 39-78 tiles per CTA, the benchmark's shape and the config-5 trace's 16-column tiles;
with 1, 2 and 4 cosets (added_bits 0-2).  The in-place forward pass reads its input as the cosets' blocks stacked in the
tensor map's last dimension.  Every case must stay on the three-launch path and match the CPU oracle in a poisoned, guarded
output buffer (test_gpu_lde_paths.run_lde_checked)."""
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_gpu_lde_paths import run_lde_checked

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def _check(gpu, f, log_h, w, added_bits):
    m = O.random_matrix(f.id, 1 << log_h, w, seed=9100 + 1000 * log_h + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("w", [4, 40, 60])
@pytest.mark.parametrize("added_bits", [0, 1, 2])
def test_producer_ring_tile_counts(gpu, f, w, added_bits, monkeypatch):
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^14 rows take the TMA pipeline by default
    _check(gpu, f, 14, w, added_bits)


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("w,added_bits", [(100, 0), (100, 2), (16, 1)])
def test_producer_ring_full_height(gpu, f, w, added_bits):
    _check(gpu, f, 20, w, added_bits)
