"""The block-row order of the coset LDE's tile-major scratch (csrc/ntt.cu: tile_block_row, ntt_lde_mid_kernel<F, R, true, CT, PROD>).

On the tile-major plan the fused middle pass stores forward step 2's results from registers, register b of item j to block row
b * 2^Q2 + j, and the gathering band pass reads block row tile_block_row(i) for band i.  The order differs between even r (one
step-2 item per thread, Q1 = Q2) and odd r (two items per thread, Q2 = Q1 + 1), and between the producer-warp instances and the
runtime-width instance at r = 10 (12-column tiles: 72 columns), which loads its own tiles.  At 2^14 rows (r = 7) each width is
checked against the CPU oracle; at 2^16, 2^18 and 2^20 rows (r = 8, 9, 10) the result must be bit-identical to the dense layout on
the band pass and on the tile kernel, written over poisoned, guarded outputs after a dirty call."""
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_gpu_lde_band import _lde_poisoned
from test_gpu_lde_gather import _check_body, _gathers
from test_gpu_lde_paths import G, run_lde_checked

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


# 64 / 100: the producer-warp instances with 16- and 20-column tiles; 72: 12-column tiles (the runtime-width instance)
@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [64, 100, 72])
@pytest.mark.parametrize("added_bits", [0, 1, 2])
def test_tile_rows_small_match_oracle(gpu, f, w, added_bits, monkeypatch):
    assert _gathers(14, w)
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^14 rows take the TMA pipeline by default; the three-launch path needs it off
    m = O.random_matrix(f.id, 1 << 14, w, seed=7300 + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)


# r = 8, 9, 10; four cosets (added_bits 2) on each; 2^20 x 72 runs the fused pass without a producer warp
SHAPES = [(16, 64, 1), (16, 72, 2), (16, 100, 0), (18, 72, 1), (18, 100, 2), (20, 72, 1), (20, 72, 2), (20, 100, 2), (20, 64, 0)]


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w,added_bits", SHAPES)
def test_tile_rows_match_dense_layout(gpu, f, log_h, w, added_bits, monkeypatch):
    assert _gathers(log_h, w)
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    h = 1 << log_h
    gen = torch.Generator(device="cuda").manual_seed(53 * log_h + w + 1000 * added_bits)
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


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_tile_rows_back_to_back(gpu, f):
    # ten LDEs on one stream with no synchronisation, alternating the producer-warp and the runtime-width fused instance over the
    # same scratch, each checked against a synchronised LDE of its own input
    calls = [(100, 1), (72, 1)] * 5
    h = 1 << 20
    gpu._use_torch_stream()
    gen = torch.Generator(device="cuda").manual_seed(8383 + f.id)
    xs, outs = [], []
    for w, added_bits in calls:
        xs.append(torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen))
        outs.append(torch.full(((h << added_bits) * w,), -1, dtype=torch.int32, device="cuda"))
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, xs[-1].data_ptr(), h, w, added_bits, f.generator, outs[-1].data_ptr(), 1))
    torch.cuda.synchronize()
    for i, ((w, added_bits), x, out) in enumerate(zip(calls, xs, outs)):
        want = torch.full_like(out, -1)
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, want.data_ptr(), 1))
        torch.cuda.synchronize()
        bad = out != want
        if bool(bad.any()):
            j = int(torch.nonzero(bad)[0])
            pytest.fail(f"{f.name} LDE 2^20 x {w}, added_bits {added_bits}, call {i} of {len(calls)}: {int(bad.sum())} words differ "
                        f"from a synchronised call; first at row {j // w}, column {j % w}")
