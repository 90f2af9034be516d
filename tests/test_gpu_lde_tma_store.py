"""The three-launch coset LDE (inverse pass 1, the fused middle pass, forward pass 2; csrc/ntt.cu coset_lde_impl) stores every
tile of its first two launches with one TMA tensor copy out of its padded shared-memory layout.  Checked against the CPU oracle for both fields at
2^14-2^18 rows (P3GPU_NTT_PIPE=0, 7 to 9 layers per pass) and at 2^20 rows (the default kernel choice), for 20-column tiles
(100), ragged 16-column tiles (44 = 16 + 16 + 12), a 24-column pass tile (24; 12-column fused tiles), one 16-column tile and
a narrow runtime-width tile (8), with 0-2 added bits.  A call that takes exactly three launches is the TMA-store path: every
other LDE plan takes four or more.  The output goes into a poisoned, guarded buffer after a dirty call on other data
(test_gpu_lde_paths.run_lde_checked), so a tile whose store is dropped cannot pass on data left by an earlier call."""
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
    m = O.random_matrix(f.id, 1 << log_h, w, seed=7000 + 1000 * log_h + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)   # three launches: the TMA-store path


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("log_h", [14, 16, 18])
@pytest.mark.parametrize("w", [100, 44, 24, 16, 8])
@pytest.mark.parametrize("added_bits", [0, 1, 2])
def test_tma_store_lde_matches_oracle(gpu, f, log_h, w, added_bits, monkeypatch):
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    _check(gpu, f, log_h, w, added_bits)


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("w,added_bits", [(100, 1), (44, 2), (8, 0)])
def test_tma_store_lde_full_height_matches_oracle(gpu, f, w, added_bits):
    _check(gpu, f, 20, w, added_bits)
