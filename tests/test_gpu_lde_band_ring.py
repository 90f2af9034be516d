"""Back-to-back band-pass LDEs on one stream (csrc/ntt.cu: ntt_band_pass_kernel, 8-CTA clusters, 3-slot ring).

Ten LDEs of different seeded inputs are enqueued on one stream with no synchronisation between them, each into its own output,
so that a launch starts while the previous one's last bulk stores may still be draining.  Each output must be bit-identical to
the same LDE on the tile kernel (P3GPU_NTT_BAND=0).  This catches ring state, mbarrier phases or undrained stores that leak
from one launch into the next, which a single call per shape cannot show."""
import pytest
import torch

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu

pytestmark = pytest.mark.gpu
N_LDES = 10


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def _lde(gpu, f, x, h, w, added_bits, out):
    _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), h, w, added_bits, f.generator, out.data_ptr(), 1))


@pytest.mark.parametrize("f", [BabyBear, KoalaBear], ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w,added_bits", [(20, 100, 1), (18, 200, 2)])
def test_band_pass_back_to_back(gpu, f, log_h, w, added_bits, monkeypatch):
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")   # 2^18 rows take the TMA pipeline by default; the band pass needs it off
    h, H = 1 << log_h, 1 << (log_h + added_bits)
    gpu._use_torch_stream()
    gen = torch.Generator(device="cuda").manual_seed(4242 + log_h + w + f.id)
    xs, outs = [], []
    for _ in range(N_LDES):
        xs.append(torch.randint(0, f.P, (h * w,), dtype=torch.int32, device="cuda", generator=gen))
        outs.append(torch.full((H * w,), -1, dtype=torch.int32, device="cuda"))
        _lde(gpu, f, xs[-1], h, w, added_bits, outs[-1])
    torch.cuda.synchronize()
    monkeypatch.setenv("P3GPU_NTT_BAND", "0")
    want = torch.empty((H * w,), dtype=torch.int32, device="cuda")
    for i, (x, out) in enumerate(zip(xs, outs)):
        _lde(gpu, f, x, h, w, added_bits, want)
        torch.cuda.synchronize()
        bad = out != want
        if bool(bad.any()):
            j = int(torch.nonzero(bad)[0])
            pytest.fail(f"{f.name} LDE 2^{log_h} x {w}, added_bits {added_bits}, call {i} of {N_LDES}: {int(bad.sum())} words differ "
                        f"from the tile kernel; first at row {j // w}, column {j % w}")
