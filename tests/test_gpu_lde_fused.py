"""The two-pass coset LDE with bit-reversed rows runs as three launches: inverse pass 1, one fused pass (inverse layers [r, 2r)
and every coset's forward layers [0, r), csrc/ntt.cu ntt_lde_mid_kernel) and forward pass 2.  At 2^20 rows the cp.async kernel
takes it by default; P3GPU_NTT_PIPE=0 puts every two-pass height on it, so the whole output can be checked against the CPU
oracle at 2^14-2^18 (7 to 9 layers per pass).  Widths: 20-column tiles (100), ragged 16-column tiles (44 = 16 + 16 + 12),
one 16-column tile, narrow runtime-width tiles (8; 24 = 12 + 12) and a width without 16-byte row segments (6), which keeps the
four-launch path.  Each case asserts its launch count and writes into a poisoned, guarded buffer after a dirty call on other
data (test_gpu_lde_paths.run_lde_checked)."""
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


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("log_h", [14, 16, 18])
@pytest.mark.parametrize("w", [100, 44, 24, 16, 8, 6])
@pytest.mark.parametrize("added_bits", [0, 1, 2])
def test_two_pass_lde_on_cp_async_kernel_matches_oracle(gpu, f, log_h, w, added_bits, monkeypatch):
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    m = O.random_matrix(f.id, 1 << log_h, w, seed=1000 * log_h + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=4 if w % 4 else 3)   # w = 6: no 16-byte rows, four launches
