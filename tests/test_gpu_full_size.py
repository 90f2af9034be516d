"""GPU parity at the BASELINE.json config 4 and config 5 SHAPES (the sizes bench.py times), through the C ABI.

The CPU oracle cannot redo 10 GB of LDE + Merkle in a unit test, so each test checks, at the full shape:
  * every word of the resident LDE against tests/ntt_reference.py on the device, and the launch count of the commit's LDE (a
    dispatch change that moves it to another path fails here);
  * spot leaf digests against the oracle's sponge over the full-width row;
  * the left-most 2^12-row sub-tree against an oracle tree over those rows (sub-tree consistency);
  * a checksum of checksums: the cap recomputed on the CPU from a middle digest layer;
  * for config 4 the FRI commit phase on the full 2^23-long codeword against the oracle, round by round.
"""
import numpy as np
import pytest
import torch

from oracle import p3_oracle as O
import ntt_reference as R
from test_gpu_lde_paths import check_matrix

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from plonky3_b200.poseidon2 import default_poseidon2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    g = default_gpu(0)
    for f in (BabyBear, KoalaBear):
        for w in (16, 24):
            default_poseidon2(f, w).upload(g)
    return g


def host(t):
    return t.cpu().numpy().view(np.uint32)


def _cap_from_layer(ohs, layer, cap_len):
    lay = np.array(layer)
    while lay.shape[0] > cap_len:
        lay = np.array([O.compress(ohs, lay[2 * i], lay[2 * i + 1]) for i in range(lay.shape[0] // 2)])
    return lay


def _check_commit(gpu, f, hash_kind, ohs, log_h, w, ntt_launches, cap_height):
    """ntt_launches: the launches of the commit's LDE, which identify its path.  They are counted as the commit's launches less
    those of merkle_commit over the resident LDE: this assumes that p3gpu_pcs_commit_dev hashes with the same call
    (hash_merkle_commit on one matrix), so a change to either one that makes their launches differ shows as a wrong LDE count
    here."""
    h = 1 << log_h
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    x = torch.randint(0, f.P, (h, w), device="cuda", dtype=torch.int32, generator=g)
    gpu.coset_lde_batch(f.id, x[:, :8].contiguous(), 1, f.generator)        # the twiddle heaps, so that none is built below
    n0 = gpu.launches
    lde, layers = gpu.pcs_commit(f.id, hash_kind, x, 1)                      # TwoAdicFriPcs::commit: LDE + MMCS, resident
    n1 = gpu.launches
    gpu.merkle_commit(f.id, hash_kind, [lde])
    n = (n1 - n0) - (gpu.launches - n1)
    assert n == ntt_launches, f"the commit's LDE took {n} launches instead of {ntt_launches}: it left the path it pins"
    H = 2 * h
    assert tuple(lde.shape) == (H, w)
    assert [int(l.shape[0]) for l in layers] == [H >> k for k in range(log_h + 2)]
    # the whole LDE against the reference, column chunk by column chunk on the device
    check_matrix(f, lde, lambda c0, c1: R.coset_lde(f, x[:, c0:c1], 1, f.generator), lambda row, col: f"coset {row >> log_h}",
                 f"{f.name} commit LDE 2^{log_h} x {w}")
    del x
    # spot leaf digests over the full-width row
    for r in (0, 1, 54321, H // 2, H - 1):
        assert np.array_equal(host(layers[0][r:r + 1])[0], O.hash_row(ohs, host(lde[r:r + 1])[0])), r
    # left-most 2^12-row sub-tree: its root is node 0 of layer 12
    sub = O.merkle_tree(ohs, [host(lde[: 1 << 12].contiguous())])
    for k in range(13):
        assert np.array_equal(sub[k], host(layers[k][: (1 << 12) >> k].contiguous())), k
    # cap recomputed from a middle layer on the CPU
    nl = len(layers)
    cap = host(layers[nl - 1 - cap_height][: 1 << cap_height].contiguous())
    mid = host(layers[nl - 1 - 11].contiguous())                            # 2^11 nodes
    assert np.array_equal(_cap_from_layer(ohs, mid, 1 << cap_height), cap)
    return lde, layers


def test_config4_pcs_commit_keccak_babybear_2_22_x_300(gpu):
    """BASELINE config 4: BabyBear 2^22 x 300, blowup 2, SerializingHasher<PaddingFreeSponge<KeccakF,25,17,4>> leaves
    (9 permutations per row), CompressionFunctionFromHasher nodes, cap_height 3."""
    f = BabyBear
    # the LDE runs on the tiled pipeline (8 + 7 + 7 layers: six launches per chunk) in 64-column chunks: columns 0-63, ..., 256-299
    lde, layers = _check_commit(gpu, f, _lib.HASH_KECCAK, O.keccak_hasher(), 22, 300, 6 * 5, 3)
    del lde, layers
    torch.cuda.empty_cache()


def test_config4_fri_commit_phase_keccak_babybear_2_23(gpu):
    """BASELINE config 4, FRI part: commit phase on a 2^23-long EF4 codeword, arities [3]*7 + [1], Keccak MMCS, cap 3,
    fixed betas — every round cap and the final value against the oracle."""
    f = BabyBear
    ohs = O.keccak_hasher()
    vec = O.random_matrix(f.id, 1 << 23, 4, seed=5)
    betas = O.random_matrix(f.id, 10, 4, seed=6)
    ocaps, oar, ofinal = O.commit_phase(f.id, ohs, 3, vec, 1, 0, 3, betas)
    assert oar == [3] * 7 + [1]
    v = torch.from_numpy(vec.view(np.int32)).cuda()
    caps, las, final = gpu.fri_commit_phase(f.id, _lib.HASH_KECCAK, v, 1, 0, 3, 3, betas)
    assert las == oar
    for a, b in zip(caps, ocaps):
        assert np.array_equal(a, b)
    assert np.array_equal(final, ofinal)


def test_config5_pcs_commit_poseidon2_koalabear_2_20_x_1312(gpu):
    """BASELINE config 5 trace commit: KoalaBear 2^20 x 1312, blowup 2, PaddingFreeSponge<Perm24,24,16,8> leaves (82
    permutations per row), TruncatedPermutation<Perm16> nodes, cap_height 3.  At this height the LDE runs on the cp.async
    kernel's three-launch path with 16-column tiles; the tiled pipeline's driver runs 128-column chunks here (10 x 128 + 32,
    four launches each: next test)."""
    _config5_commit(gpu, 3)


def _config5_commit(gpu, ntt_launches):
    f = KoalaBear
    ohs = O.poseidon2_hasher(O.default_perm(f.id, 24), O.default_perm(f.id, 16))
    lde, layers = _check_commit(gpu, f, _lib.HASH_POSEIDON2_W24, ohs, 20, 1312, ntt_launches, 3)
    del layers
    torch.cuda.empty_cache()
    del lde
    torch.cuda.empty_cache()


def test_config5_pcs_commit_on_the_tiled_pipeline(gpu, monkeypatch):
    """The same commit with P3GPU_NTT_PIPE=1: the LDE on the TMA pipeline with column-tile-major intermediates, in chunks."""
    monkeypatch.setenv("P3GPU_NTT_PIPE", "1")
    _config5_commit(gpu, 4 * 11)


def test_config5_fri_commit_phase_poseidon2_koalabear_2_21(gpu):
    """BASELINE config 5, FRI part: 2^21-long codeword, arities [3]*6 + [2], Poseidon2 MMCS (width-24 leaves), cap 3."""
    f = KoalaBear
    ohs = O.poseidon2_hasher(O.default_perm(f.id, 24), O.default_perm(f.id, 16))
    vec = O.random_matrix(f.id, 1 << 21, 4, seed=7)
    betas = O.random_matrix(f.id, 10, 4, seed=8)
    ocaps, oar, ofinal = O.commit_phase(f.id, ohs, 3, vec, 1, 0, 3, betas)
    assert oar == [3] * 6 + [2]
    v = torch.from_numpy(vec.view(np.int32)).cuda()
    caps, las, final = gpu.fri_commit_phase(f.id, _lib.HASH_POSEIDON2_W24, v, 1, 0, 3, 3, betas)
    assert las == oar
    for a, b in zip(caps, ocaps):
        assert np.array_equal(a, b)
    assert np.array_equal(final, ofinal)
