"""GPU parity tests: every hot-path entry point of libp3gpu (called through the C ABI via plonky3_b200) against the CPU
oracle on the same seeded inputs — bit-exact — plus size-independent properties at the BASELINE.json sizes.
Run on an H100 with `pytest -m gpu`."""
import json
import pathlib

import numpy as np
import pytest
import torch

from oracle import p3_oracle as O
import fixture_replay as FR
import ntt_reference as R
from test_gpu_lde_paths import check_matrix

import plonky3_b200 as P
from plonky3_b200 import _lib
from plonky3_b200.dft import Radix2DitParallel, reverse_matrix_index_bits
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriFolding, TwoAdicFriPcs, commit_phase
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import Poseidon2, default_poseidon2

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).resolve().parent / "golden"
FIELDS = [BabyBear, KoalaBear]


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


# ------------------------------------------------------------------------------------------ config 1
def test_config1_forward_ntt_babybear_2_16(gpu):
    """BASELINE config 1: Radix2DitParallel forward NTT, BabyBear, 2^16 x 1, bit-exact; plus the edge inputs."""
    f = BabyBear
    dft = Radix2DitParallel(f, gpu)
    h = 1 << 16
    m = O.random_matrix(f.id, h, 1, seed=1)
    assert np.array_equal(dft.dft_batch(m), O.dft_batch(f.id, m))
    assert np.array_equal(dft.dft(m.ravel()), O.dft_batch(f.id, m).ravel())
    zero = np.zeros((h, 1), dtype=np.uint32)
    assert not dft.dft_batch(zero).any()
    delta = zero.copy(); delta[0, 0] = f.ONE
    assert (dft.dft_batch(delta) == f.ONE).all()
    allm1 = np.full((h, 1), f.to_monty(f.P - 1), dtype=np.uint32)
    assert np.array_equal(dft.dft_batch(allm1), O.dft_batch(f.id, allm1))


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w", [(0, 3), (1, 1), (2, 5), (3, 17), (5, 4), (7, 33), (9, 100), (10, 7), (11, 36), (12, 3), (13, 20), (15, 2),
                                     (10, 33), (10, 45), (9, 21), (8, 24), (10, 25), (7, 48), (10, 52)])
def test_dft_family_matches_oracle(gpu, f, log_h, w):
    # dft/tests/testing.rs:298-378: dft / idft / coset_dft / coset_idft agree with the definition for many shapes
    dft = Radix2DitParallel(f, gpu)
    m = O.random_matrix(f.id, 1 << log_h, w, seed=100 * log_h + w)
    shift = f.to_monty(0x2345678 + log_h)
    assert np.array_equal(dft.dft_batch(m), O.dft_batch(f.id, m))
    assert np.array_equal(dft.idft_batch(m), O.idft_batch(f.id, m))
    assert np.array_equal(dft.coset_dft_batch(m, shift), O.coset_dft_batch(f.id, m, shift))
    assert np.array_equal(dft.coset_idft_batch(m, shift), O.coset_idft_batch(f.id, m, shift))
    # device-resident path gives the same answer as the host-pointer path
    assert np.array_equal(host(dft.dft_batch(dev(m))), O.dft_batch(f.id, m))


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_small_dft_vs_naive_definition(gpu, f):
    # field-testing/src/dft_testing.rs:307-405 (h <= 16, w = 3 vs NaiveDft)
    dft = Radix2DitParallel(f, gpu)
    for log_h in range(0, 5):
        m = O.random_matrix(f.id, 1 << log_h, 3, seed=log_h)
        assert np.array_equal(dft.dft_batch(m), O.naive_dft(f.id, m))


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h,w,added_bits", [(0, 2, 1), (1, 3, 2), (4, 5, 0), (4, 5, 1), (6, 9, 3), (10, 100, 1), (12, 37, 1), (13, 8, 2), (14, 4, 1), (10, 33, 1), (9, 45, 2),
                                                  (12, 100, 1), (16, 40, 2), (14, 128, 1), (13, 12, 1), (15, 8, 0)])
def test_coset_lde_matches_oracle(gpu, f, log_h, w, added_bits):
    # traits.rs:227-259 + radix_2_dit_parallel.rs:181-246: values AND memory layout (bit-reversed rows)
    dft = Radix2DitParallel(f, gpu)
    m = O.random_matrix(f.id, 1 << log_h, w, seed=7 * log_h + w)
    shift = f.generator
    view = dft.coset_lde_batch(m, added_bits, shift)
    assert np.array_equal(view.bit_reverse_rows(), O.coset_lde_batch(f.id, m, added_bits, shift, bitrev_out=True))
    assert np.array_equal(view.to_row_major_matrix(), O.coset_lde_batch(f.id, m, added_bits, shift, bitrev_out=False))
    nat = gpu.coset_lde_batch(f.id, m, added_bits, shift, bitrev_rows=False)
    assert np.array_equal(nat, O.coset_lde_batch(f.id, m, added_bits, shift, bitrev_out=False))
    assert np.array_equal(host(dft.coset_lde_batch(dev(m), added_bits, shift).bit_reverse_rows()), view.bit_reverse_rows())
    assert np.array_equal(dft.lde_batch(m, added_bits).bit_reverse_rows(), O.coset_lde_batch(f.id, m, added_bits, f.ONE, True))


@pytest.mark.parametrize("f,log_h,w", [(BabyBear, 22, 3), (KoalaBear, 21, 4), (BabyBear, 23, 1), (KoalaBear, 17, 24), (BabyBear, 19, 20)])
def test_large_heights_three_pass_plans(gpu, f, log_h, w):
    # heights above 2^20 run as three passes (7+7+7, 8+7+7, 8+8+7 layers); BASELINE config 4 is 2^22 rows
    dft = Radix2DitParallel(f, gpu)
    m = O.random_matrix(f.id, 1 << log_h, w, seed=log_h)
    assert np.array_equal(dft.dft_batch(m), O.dft_batch(f.id, m))
    got = dft.coset_lde_batch(dev(m), 1, f.generator).bit_reverse_rows()
    assert np.array_equal(host(got), O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True))


@pytest.mark.parametrize("f,log_h,w,added_bits,chunk", [(KoalaBear, 13, 52, 1, 16), (BabyBear, 12, 100, 2, 24), (KoalaBear, 21, 8, 1, 0), (BabyBear, 19, 12, 1, 8)])
def test_coset_lde_tiled_intermediates(gpu, f, log_h, w, added_bits, chunk, monkeypatch):
    # the pipelined LDE keeps its intermediates column-tile-major and walks wide matrices in column chunks (csrc/ntt.cu
    # lde_tiled_impl); P3GPU_NTT_CHUNK forces small chunks so that the chunk loop and ragged last tiles are exercised.
    # Dense LDEs take the cp.async kernel by default: P3GPU_NTT_PIPE=1 puts this one on the pipeline.
    monkeypatch.setenv("P3GPU_NTT_PIPE", "1")
    if chunk:
        monkeypatch.setenv("P3GPU_NTT_CHUNK", str(chunk))
    dft = Radix2DitParallel(f, gpu)
    m = O.random_matrix(f.id, 1 << log_h, w, seed=3 * log_h + w)
    got = dft.coset_lde_batch(dev(m), added_bits, f.generator).bit_reverse_rows()
    assert np.array_equal(host(got), O.coset_lde_batch(f.id, m, added_bits, f.generator, bitrev_out=True))


@pytest.mark.parametrize("f,log_h,w,pipelined", [(BabyBear, 21, 200, 24), (KoalaBear, 22, 72, 12)], ids=["f0-21-200", "f1-22-72"])
def test_lde_many_small_tiles_pipelined_vs_cp_async_kernels(gpu, f, log_h, w, pipelined, monkeypatch):
    # three-pass plans have 128/256-row tiles that are processed faster than HBM latency varies: the regime in which a consumer
    # group of the pipelined kernel can run ahead of an in-flight load (mbarrier phase handling, csrc/ntt.cu).  The cp.async
    # kernel's result (six launches: the inverse and the forward network, three passes each) is checked word for word against
    # the reference transform on the device, and the TMA pipeline's (six launches per 64-column chunk: 3 x 64 + 8 columns at
    # 2^21 x 200, 64 + 8 at 2^22 x 72) must equal it bit for bit.  Each repeat writes into an output filled with 0xFFFFFFFF
    # (never canonical): a tile whose store is dropped cannot pass on the previous repeat's result, which the caching allocator
    # would otherwise hand back in the same block.
    x = torch.randint(0, f.P, (1 << log_h, w), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(log_h))
    monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    gpu.coset_lde_batch(f.id, x, 1, f.generator)                                    # twiddle heaps
    n0 = gpu.launches
    want = gpu.coset_lde_batch(f.id, x, 1, f.generator)
    assert gpu.launches - n0 == 6, "cp.async kernel: the case left the path it pins"
    check_matrix(f, want, lambda c0, c1: R.coset_lde(f, x[:, c0:c1], 1, f.generator), lambda row, col: f"coset {row >> log_h}",
                 f"{f.name} LDE 2^{log_h} x {w} on the cp.async kernel")
    monkeypatch.setenv("P3GPU_NTT_PIPE", "1")
    for _ in range(3):
        got = torch.full_like(want, -1)
        gpu._use_torch_stream()
        n0 = gpu.launches
        _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr(), x.shape[0], w, 1, f.generator, got.data_ptr(), 1))
        assert gpu.launches - n0 == pipelined, "TMA pipeline: the case left the path it pins"
        assert torch.equal(got, want)
        del got


def test_dft_shape_errors(gpu):
    # the reference panics in log2_strict_usize on non power-of-two heights; the C ABI returns P3GPU_EINVAL
    with pytest.raises(P.P3GpuError, match="power of two"):
        gpu.dft_batch(0, _lib.DFT, np.zeros((6, 2), dtype=np.uint32))
    # 2^24 rows + 1 added bit exceeds KoalaBear's two-adicity (24): rejected before any memory is touched
    rc = gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, KoalaBear.id, 256, 1 << 24, 1, 1, KoalaBear.ONE, 512, 1)
    assert rc == -1 and b"two-adicity" in gpu.L.p3gpu_last_error()
    with pytest.raises(ValueError):
        Radix2DitParallel(KoalaBear, gpu).dft_batch(np.zeros((12, 1), dtype=np.uint32))


# ------------------------------------------------------------------------------------------ hashing
def test_poseidon2_kats_on_gpu(gpu):
    # koala-bear/src/poseidon2.rs:614-653, baby-bear/src/poseidon2.rs:599-639
    kats = json.loads((GOLD / "poseidon2_kat.json").read_text())
    for f in FIELDS:
        for w in (16, 24):
            k = kats[f"{f.name}_{w}"]
            pm = default_poseidon2(f, w)
            out = pm.permute(gpu, f.to_monty_array(k["input"]).reshape(1, w))
            assert f.from_monty_array(out[0]).tolist() == k["expected"]


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [16, 24])
def test_poseidon2_random_states(gpu, f, w):
    pm = default_poseidon2(f, w)
    st = O.random_matrix(f.id, 300, w, seed=w)
    st[0] = 0; st[1] = f.P - 1
    out = pm.permute(gpu, st)
    opm = O.default_perm(f.id, w)
    for i in range(0, 300, 7):
        assert np.array_equal(out[i], O.poseidon2_permute(opm, st[i]))


def test_keccak_f_on_gpu(gpu):
    rng = np.random.default_rng(3)
    st = rng.integers(0, 1 << 63, size=(70, 25), dtype=np.uint64) * 2 + rng.integers(0, 2, size=(70, 25), dtype=np.uint64)
    st[0] = 0
    out = gpu.keccak_f(st)
    for i in range(70):
        assert np.array_equal(out[i], O.keccak_f(st[i]))


def _mmcs_pair(f, kind, gpu, cap_height=0):
    """(GPU mmcs, oracle hasher) for one of the three hash configurations."""
    if kind == "keccak":
        return MerkleTreeMmcs.keccak(f, cap_height, gpu), O.keccak_hasher()
    p16 = default_poseidon2(f, 16)
    if kind == "p2w16":
        return MerkleTreeMmcs.poseidon2(p16, None, cap_height, gpu), O.poseidon2_hasher(O.default_perm(f.id, 16), O.default_perm(f.id, 16))
    return MerkleTreeMmcs.poseidon2(p16, default_poseidon2(f, 24), cap_height, gpu), O.poseidon2_hasher(O.default_perm(f.id, 24), O.default_perm(f.id, 16))


def _check_tree(tree, olayers):
    assert len(tree.digest_layers) == len(olayers)
    for a, b in zip(tree.digest_layers, olayers):
        a = host(a) if torch.is_tensor(a) else a
        assert np.array_equal(a, b)


@pytest.mark.parametrize("kind", ["p2w16", "p2w24", "keccak"])
@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_merkle_single_matrix_widths(gpu, f, kind):
    # widths below / equal / above the sponge rate, odd widths (Keccak pair packing), wide rows
    mmcs, ohs = _mmcs_pair(f, kind, gpu)
    for h, w in [(1, 5), (2, 8), (8, 1), (16, 16), (32, 17), (64, 33), (128, 34), (256, 35), (512, 100), (1024, 7)]:
        m = O.random_matrix(f.id, h, w, seed=h + w)
        cap, tree = mmcs.commit([m])
        ol = O.merkle_tree(ohs, [m])
        _check_tree(tree, ol)
        assert np.array_equal(cap, O.merkle_cap(ol, 0))
        cap_d, tree_d = mmcs.commit([dev(m)])
        _check_tree(tree_d, ol)


@pytest.mark.parametrize("kind", ["p2w16", "p2w24", "keccak"])
def test_merkle_mixed_heights_caps_and_padding(gpu, kind):
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, kind, gpu, cap_height=2)
    mats = [O.random_matrix(f.id, 64, 3, seed=1), O.random_matrix(f.id, 256, 9, seed=2), O.random_matrix(f.id, 256, 5, seed=3),
            O.random_matrix(f.id, 8, 21, seed=4), O.random_matrix(f.id, 64, 2, seed=5)]
    cap, tree = mmcs.commit(mats)
    ol = O.merkle_tree(ohs, mats)
    _check_tree(tree, ol)
    assert np.array_equal(cap, O.merkle_cap(ol, 2)) and cap.shape == (4, 8)
    # non power-of-two heights on the ladder: 21 -> 11 -> 6 (merkle_tree.rs:652-711 padding with the zero digest)
    mats = [O.random_matrix(f.id, 21, 4, seed=6), O.random_matrix(f.id, 11, 3, seed=7), O.random_matrix(f.id, 6, 2, seed=8)]
    cap, tree = mmcs.commit(mats)
    _check_tree(tree, O.merkle_tree(ohs, mats))
    # open_batch: rows and sibling path (mmcs/batch.rs:75-121)
    openings, proof = mmcs.open_batch(13, tree)
    assert np.array_equal(openings[0], mats[0][13]) and np.array_equal(openings[1], mats[1][6]) and np.array_equal(openings[2], mats[2][3])
    # heights off the ladder are rejected (mmcs/geometry.rs:83-124)
    with pytest.raises(P.P3GpuError, match="incompatible"):
        mmcs.commit([O.random_matrix(f.id, 8, 1), O.random_matrix(f.id, 3, 1)])
    with pytest.raises(P.P3GpuError):
        mmcs.commit([])


# ------------------------------------------------------------------------------------------ FRI
@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_arity", [1, 2, 3, 4])
def test_fold_matrix_matches_oracle(gpu, f, log_arity):
    fold = TwoAdicFriFolding(f, gpu)
    for log_len in (log_arity, log_arity + 1, 9, 13):
        v = O.random_matrix(f.id, 1 << log_len, 4, seed=log_len)
        beta = O.random_matrix(f.id, 1, 4, seed=99)[0]
        exp = O.fold_matrix(f.id, v, log_arity, beta)
        assert np.array_equal(fold.fold_matrix(beta, log_arity, v), exp)
        assert np.array_equal(host(fold.fold_matrix(beta, log_arity, dev(v))), exp)


class FixedBetaChallenger:
    """Transcript stand-in for parity tests: records caps, returns a fixed beta list (PoW bits = 0)."""

    def __init__(self, betas): self.betas = list(betas); self.caps = []; self.final = None
    def observe_cap(self, cap): self.caps.append(np.array(cap))
    def grind(self, bits): assert bits == 0; return 0
    def sample_algebra_element(self): return self.betas.pop(0)
    def observe_algebra_slice(self, v): self.final = np.array(v)


@pytest.mark.parametrize("kind,f", [("p2w16", BabyBear), ("p2w24", KoalaBear), ("keccak", BabyBear)])
def test_commit_phase_matches_oracle(gpu, kind, f):
    # fri/src/prover.rs:192-286 with benchmark parameters (blowup 2, max arity 8, no commit PoW), cap_height 3
    mmcs, ohs = _mmcs_pair(f, kind, gpu, cap_height=3)
    params = FriParameters.new_benchmark_high_arity(mmcs)
    log_len = 12
    vec = O.random_matrix(f.id, 1 << log_len, 4, seed=5)
    betas = O.random_matrix(f.id, 8, 4, seed=6)
    ocaps, oar, ofinal = O.commit_phase(f.id, ohs, 3, vec, params.log_blowup, params.log_final_poly_len, params.max_log_arity, betas)
    ch = FixedBetaChallenger(betas)
    res = commit_phase(TwoAdicFriFolding(f, gpu), params, [dev(vec)], ch, Radix2DitParallel(f, gpu))
    assert res.log_arities == oar == [3, 3, 3, 2]
    for a, b in zip(res.commits, ocaps):
        assert np.array_equal(a, b)
    assert np.array_equal(res.final_poly, ofinal[:1])
    # single-call device driver
    caps, las, final = gpu.fri_commit_phase(f.id, mmcs.hash_kind, dev(vec), 1, 0, 3, 3, betas)
    assert las == oar and all(np.array_equal(a, b) for a, b in zip(caps, ocaps)) and np.array_equal(final, ofinal)


def test_commit_phase_with_two_input_heights(gpu):
    # fri/src/prover.rs:258-265: a shorter input is rolled in as folded += beta^arity * input; the arity schedule stops at
    # the next input's height (config.rs:180-207)
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, "p2w16", gpu, cap_height=1)
    params = FriParameters.new_benchmark_high_arity(mmcs)
    v0, v1 = O.random_matrix(f.id, 1 << 10, 4, seed=1), O.random_matrix(f.id, 1 << 8, 4, seed=2)
    betas = O.random_matrix(f.id, 8, 4, seed=3)
    ocaps, oar, ofinal = O.commit_phase(f.id, ohs, 1, [v0, v1], 1, 0, 3, betas)
    assert oar[0] == 2
    ch = FixedBetaChallenger(betas)
    res = commit_phase(TwoAdicFriFolding(f, gpu), params, [dev(v0), dev(v1)], ch, Radix2DitParallel(f, gpu))
    assert res.log_arities == oar
    assert all(np.array_equal(a, b) for a, b in zip(res.commits, ocaps))
    assert np.array_equal(res.final_poly, ofinal[:1])


def test_commit_quotient_matches_oracle(gpu):
    # Pcs::commit_quotient (commit/src/pcs/univariate.rs:98-119): split_evals -> sub-coset LDEs -> one batch commitment
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, "p2w24", gpu, cap_height=0)
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), mmcs, FriParameters.new_benchmark_high_arity(mmcs))
    log_n, chunks = 9, 2
    q = O.random_matrix(f.id, 1 << log_n, 4, seed=4)                    # evaluations over GENERATOR * H, natural order
    cap, tree = pcs.commit_quotient((f.generator, log_n), q, chunks)
    h = O.two_adic_generator(f.id, log_n)
    ldes = []
    for i in range(chunks):
        sub = np.ascontiguousarray(q[i::chunks])
        dshift = O.mul(f.id, f.generator, O.fpow(f.id, h, i))
        ldes.append(O.coset_lde_batch(f.id, sub, 1, O.mul(f.id, f.generator, O.inv(f.id, dshift)), bitrev_out=True))
    assert np.array_equal(cap, O.merkle_cap(O.merkle_tree(ohs, ldes), 0))


def test_pcs_commit_matches_oracle(gpu):
    # TwoAdicFriPcs::commit (two_adic_pcs.rs:300-324): LDE onto GENERATOR*K, bit-reversed, Poseidon2 MMCS
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, "p2w24", gpu, cap_height=3)
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), mmcs, FriParameters.new_benchmark_high_arity(mmcs))
    m = O.random_matrix(f.id, 1 << 10, 45, seed=8)
    cap, tree = pcs.commit([(pcs.natural_domain_for_degree(1 << 10), m)])
    lde = O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True)
    ol = O.merkle_tree(ohs, [lde])
    assert np.array_equal(cap, O.merkle_cap(ol, 3))
    assert np.array_equal(mmcs.get_matrices(tree)[0], lde)
    lde_d, layers = gpu.pcs_commit(f.id, mmcs.hash_kind, dev(m), 1)
    assert np.array_equal(host(lde_d), lde) and np.array_equal(host(layers[-1]), ol[-1])
    ev = pcs.get_evaluations_on_domain(tree, 0, (f.generator, 10))
    assert np.array_equal(ev.to_row_major_matrix(), O.coset_dft_batch(f.id, O.idft_batch(f.id, m), f.generator))


class GpuBackend:
    """fixture_replay backend on the GPU: every hot-path step of the proof goes through libp3gpu."""

    def __init__(self, gpu):
        rc_i, rc_t, rc_p = FR.fixture_constants()
        pm = Poseidon2.new(BabyBear, 16, rc_i, rc_t, rc_p, monty=True)
        self.mmcs = MerkleTreeMmcs.poseidon2(pm, None, 0, gpu)
        self.dft = Radix2DitParallel(BabyBear, gpu)
        self.folding = TwoAdicFriFolding(BabyBear, gpu)

    def lde(self, mat, added_bits, shift): return self.dft.coset_lde_batch(mat, added_bits, shift).bit_reverse_rows()
    def commit(self, mats): return self.mmcs.commit(mats)[0]
    def fold(self, vec, log_arity, beta): return self.folding.fold_matrix(beta, log_arity, vec)
    def commit_data(self, mats): return self.mmcs.commit([dev(m) for m in mats])            # device-resident prover data
    def open_multi(self, data, indices): return self.mmcs.open_multi_batch(indices, data)   # csrc/query.cu gathers


class GpuOpenBackend(GpuBackend):
    """Adds TwoAdicFriPcs::open's pre-FRI part on the GPU (inverse denominators, interpolation, alpha compression, quotients)."""

    def open(self, rounds, challenger, log_blowup):
        from plonky3_b200.merkle_tree import MerkleTree
        mmcs = self.mmcs
        pcs = TwoAdicFriPcs(self.dft, mmcs, FriParameters(log_blowup, 2, 1, 2, 1, 1, mmcs))
        data = [(MerkleTree([dev(m) for m in mats], []), points) for mats, points in rounds]
        opened, fri_inputs = pcs.open_values_and_fri_inputs(data, challenger)
        return opened, [host(v) for v in fri_inputs]


def test_fixture_replay_with_gpu_open(gpu):
    """The committed proof is reproduced with LDE, Merkle, `open` (interpolation + reduced openings) and FRI fold on the GPU."""
    gold = json.loads((GOLD / "uni_stark_two_adic_v1.json").read_text())
    got = FR.replay(GpuOpenBackend(gpu))
    for k, v in got.items():
        assert v == gold[k], k


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_open_primitives_match_oracle(gpu, f):
    # compute_inverse_denominators, columnwise_dot_product, rowwise dot with alpha powers, quotient accumulation
    z = O.random_matrix(f.id, 1, 4, seed=21)[0]; alpha = O.random_matrix(f.id, 1, 4, seed=22)[0]
    zinv = O.ef_inv(f.id, z)
    for log_h in (0, 3, 11, 20):
        inv_d, adj = gpu.open_inv_denoms(f.id, log_h, z, zinv)
        exp = O.open_inv_denoms(f.id, log_h, z)
        assert np.array_equal(host(inv_d), exp)
        # compute_adjusted_weights: adj[i] = 1/(z - x_i) - 1/z, checked against the oracle on every row (small) or a row sample
        n = 1 << log_h
        rows = np.arange(n) if log_h < 6 else np.unique(np.concatenate([[0, 1, n // 2, n - 2, n - 1], np.random.default_rng(log_h).integers(0, n, 200)]))
        got = host(adj)
        for i in rows:
            assert np.array_equal(got[i], O.ef_sub(f.id, exp[i], zinv)), (log_h, int(i))
    for h, w in [(1, 1), (8, 3), (13, 4), (64, 33), (300, 100), (4096, 7), (4097, 8), (5000, 260)]:
        m = O.random_matrix(f.id, h, w, seed=h + w)
        v = O.random_matrix(f.id, h, 4, seed=h)
        scale = O.random_matrix(f.id, 1, 4, seed=9)[0]
        exp = O.columnwise_dot(f.id, m, v)
        assert np.array_equal(host(gpu.columnwise_dot(f.id, dev(m), dev(v))), exp)
        assert np.array_equal(host(gpu.columnwise_dot(f.id, dev(m), dev(v), scale)), np.array([O.ef_mul(f.id, scale, e) for e in exp]))
        r = O.rowwise_dot(f.id, m, alpha)
        assert np.array_equal(host(gpu.rowwise_dot(f.id, dev(m), alpha)), r)
        ro = O.random_matrix(f.id, h, 4, seed=3); invd = O.random_matrix(f.id, h, 4, seed=4)
        coeff = O.random_matrix(f.id, 1, 4, seed=5)[0]; yred = O.random_matrix(f.id, 1, 4, seed=6)[0]
        assert np.array_equal(host(gpu.open_reduce(f.id, dev(ro), dev(r), dev(invd), coeff, yred)), O.open_reduce(f.id, ro, r, invd, coeff, yred))


def test_open_worst_case_accumulators(gpu):
    # all-(p-1) inputs drive the lazy 64-bit accumulators of the dot-product kernels to their bound
    f = KoalaBear
    m = np.full((4096, 40), f.P - 1, dtype=np.uint32); v = np.full((4096, 4), f.P - 1, dtype=np.uint32)
    assert np.array_equal(host(gpu.columnwise_dot(f.id, dev(m), dev(v))), O.columnwise_dot(f.id, m, v))
    alpha = np.full(4, f.P - 1, dtype=np.uint32)
    assert np.array_equal(host(gpu.rowwise_dot(f.id, dev(m), alpha)), O.rowwise_dot(f.id, m, alpha))


def test_fixture_replay_on_gpu(gpu):
    """The reference's committed proof (uni_stark_two_adic_v1.postcard) is reproduced with LDE, Merkle, FRI fold and the query
    gathers on the GPU — every field, and the serialised proof byte for byte (`postcard_hex`, 1115 bytes)."""
    gold = json.loads((GOLD / "uni_stark_two_adic_v1.json").read_text())
    got = FR.replay(GpuBackend(gpu))
    assert "postcard_hex" in got and "input_openings" in got
    for k, v in got.items():
        assert v == gold[k], k


# ------------------------------------------------------------------------------------------ full-size properties
def test_config2_lde_full_size_properties(gpu):
    """BASELINE config 2 (KoalaBear 2^20 x 100, blowup 2): spot columns vs the oracle + round trip + linearity."""
    f = KoalaBear
    h, w = 1 << 20, 100
    dft = Radix2DitParallel(f, gpu)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    x = torch.randint(0, f.P, (h, w), device="cuda", dtype=torch.int32, generator=g)
    lde = dft.coset_lde_batch(x, 1, f.generator).bit_reverse_rows()
    cols = [0, 37, 99]
    xs = host(x[:, cols].contiguous())
    exp = O.coset_lde_batch(f.id, xs, 1, f.generator, bitrev_out=True)
    assert np.array_equal(host(lde[:, cols].contiguous()), exp)
    # round trip: the first h memory rows are the evaluations on GENERATOR*H (bit-reversed) -> coset iDFT gives idft(x)
    first = reverse_matrix_index_bits(lde[:h].contiguous())
    assert torch.equal(dft.coset_idft_batch(first, f.generator), dft.idft_batch(x))
    # linearity: LDE(x + y) = LDE(x) + LDE(y)
    y = torch.randint(0, f.P, (h, w), device="cuda", dtype=torch.int32, generator=g)
    s = (x.long() + y.long()) % f.P
    lde_y = dft.coset_lde_batch(y, 1, f.generator).bit_reverse_rows()
    lde_s = dft.coset_lde_batch(s.int(), 1, f.generator).bit_reverse_rows()
    assert torch.equal(lde_s.long(), (lde.long() + lde_y.long()) % f.P)


def test_config3_merkle_full_size_properties(gpu):
    """BASELINE config 3 (KoalaBear 2^22 x 100, Poseidon2-16 sponge): sub-tree consistency + spot leaves vs oracle."""
    f = KoalaBear
    h, w = 1 << 22, 100
    mmcs, ohs = _mmcs_pair(f, "p2w16", gpu)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    x = torch.randint(0, f.P, (h, w), device="cuda", dtype=torch.int32, generator=g)
    cap, tree = mmcs.commit([x])
    assert [int(l.shape[0]) for l in tree.digest_layers] == [h >> k for k in range(23)]
    for r in (0, 1, 12345, h - 1):
        assert np.array_equal(host(tree.digest_layers[0][r:r + 1])[0], O.hash_row(ohs, host(x[r:r + 1])[0]))
    # the tree over the first 2^12 rows is the left-most sub-tree: its root is node 0 of layer 12
    sub = O.merkle_tree(ohs, [host(x[: 1 << 12].contiguous())])
    assert np.array_equal(sub[-1][0], host(tree.digest_layers[12][0:1])[0])
    # a checksum of checksums: root recomputed from layer 12 on the CPU
    lay = host(tree.digest_layers[12].contiguous())
    while lay.shape[0] > 1:
        lay = np.array([O.compress(ohs, lay[2 * i], lay[2 * i + 1]) for i in range(lay.shape[0] // 2)])
    assert np.array_equal(lay[0], cap[0])


# ------------------------------------------------------------------------------------------ round-2 boundary hardening
@pytest.mark.parametrize("kind", ["p2w16", "p2w24", "keccak"])
def test_merkle_more_than_eight_matrices_per_height(gpu, kind):
    """MerkleTree::new takes any number of same-height matrices (merkle_tree.rs:131-133,312-316): 19 tall ones (mixed widths,
    one of width 0) plus 11 injected ones at half height."""
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, kind, gpu, cap_height=1)
    tall = [O.random_matrix(f.id, 64, 1 + (5 * k) % 23, seed=100 + k) for k in range(18)] + [np.zeros((64, 0), dtype=np.uint32)]
    short = [O.random_matrix(f.id, 32, 1 + (3 * k) % 7, seed=200 + k) for k in range(11)]
    mats = tall[:9] + short[:4] + tall[9:] + short[4:]          # input order is interleaved; the sort by height is stable
    olayers = O.merkle_tree(ohs, mats)
    cap, tree = mmcs.commit([dev(m) for m in mats])
    _check_tree(tree, olayers)
    cap_h, tree_h = mmcs.commit(mats)                            # host-pointer path (pooled arena)
    _check_tree(tree_h, olayers)
    assert np.array_equal(cap, cap_h)


def test_get_evaluations_on_domain_slow_path(gpu):
    """two_adic_pcs.rs:390-403: re-evaluation of a committed matrix on a foreign coset / a larger domain."""
    f = KoalaBear
    mmcs, _ = _mmcs_pair(f, "p2w16", gpu)
    dft = Radix2DitParallel(f, gpu)
    pcs = TwoAdicFriPcs(dft, mmcs, FriParameters.new_benchmark_high_arity(mmcs))
    m = O.random_matrix(f.id, 1 << 9, 12, seed=31)
    _, tree = pcs.commit([(pcs.natural_domain_for_degree(1 << 9), m)])
    coeffs = O.idft_batch(f.id, m)
    for shift, log_size in [(f.mul(f.generator, f.generator), 9), (f.ONE, 10), (f.generator, 11), (f.to_monty(7), 8)]:
        ev = pcs.get_evaluations_on_domain(tree, 0, (shift, log_size))
        size = 1 << log_size
        padded = np.zeros((size, 12), dtype=np.uint32)
        n = min(size, 1 << 9)
        padded[:n] = coeffs[:n]
        assert np.array_equal(ev.to_row_major_matrix(), O.coset_dft_batch(f.id, padded, shift)), (shift, log_size)
    dtree = pcs.commit([(pcs.natural_domain_for_degree(1 << 9), dev(m))])[1]          # device-resident leaves
    ev = pcs.get_evaluations_on_domain(dtree, 0, (f.ONE, 10))
    padded = np.zeros((1 << 10, 12), dtype=np.uint32); padded[: 1 << 9] = coeffs
    assert np.array_equal(host(ev.to_row_major_matrix()), O.coset_dft_batch(f.id, padded, f.ONE))


def test_commit_phase_final_polynomial_longer_than_one(gpu):
    """log_final_poly_len > 0: the folded vector is truncated, bit-reversed and iDFT'ed (fri/src/prover.rs:267-280)."""
    f = BabyBear
    mmcs, ohs = _mmcs_pair(f, "p2w16", gpu)
    params = FriParameters(1, 2, 1, 2, 0, 1, mmcs)                                    # blowup 2, final poly length 4, arity 2
    vec = O.random_matrix(f.id, 1 << 9, 4, seed=41)
    betas = O.random_matrix(f.id, 8, 4, seed=42)
    ocaps, oar, ofinal = O.commit_phase(f.id, ohs, 0, vec, 1, 2, 1, betas)
    ch = FixedBetaChallenger(betas)
    res = commit_phase(TwoAdicFriFolding(f, gpu), params, [dev(vec)], ch, Radix2DitParallel(f, gpu))
    assert res.log_arities == oar and all(np.array_equal(a, b) for a, b in zip(res.commits, ocaps))
    # oracle side of the final step: first 4 folded values, bit-reversed, iDFT of each of the 4 base coordinates
    fl = 4
    rev = O.reverse_matrix_index_bits(ofinal[:fl])
    exp = O.idft_batch(f.id, rev)
    assert np.array_equal(res.final_poly, exp)
    assert np.array_equal(ch.final, exp)


def test_one_context_shared_by_two_threads(gpu):
    """SURVEY 8b "Threading": the reference's objects are Clone + Sync; one p3gpu_ctx called from two host threads at once
    (its entry points serialise on the context's mutex) must give the same answers as sequential calls."""
    import threading
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, "p2w16", gpu)
    dft = Radix2DitParallel(f, gpu)
    ms = [O.random_matrix(f.id, 1 << 11, 20 + 4 * k, seed=50 + k) for k in range(4)]
    exp_lde = [O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True) for m in ms]
    exp_root = [O.merkle_tree(ohs, [m])[-1][0] for m in ms]
    errors = []

    def work(tid):
        try:
            for it in range(6):
                k = (tid + it) % 4
                if (tid + it) % 2 == 0:
                    got = dft.coset_lde_batch(ms[k], 1, f.generator).bit_reverse_rows()          # host-pointer call
                    assert np.array_equal(got, exp_lde[k]), ("lde", tid, it)
                else:
                    cap, _ = mmcs.commit([ms[k]])
                    assert np.array_equal(cap[0], exp_root[k]), ("merkle", tid, it)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ths = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for t in ths: t.start()
    for t in ths: t.join()
    assert not errors, errors


def test_stream_switch_orders_shared_scratch(gpu):
    """p3gpu_ctx_set_stream with a different stream between calls: work queued on the old stream (which uses the context's
    scratch buffers and may be generating twiddles) is ordered before the new stream's work."""
    f = BabyBear
    dft = Radix2DitParallel(f, gpu)
    m = O.random_matrix(f.id, 1 << 15, 24, seed=61)
    exp = O.coset_lde_batch(f.id, m, 2, f.to_monty(5), bitrev_out=True)
    x = dev(m)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for it in range(6):
        with torch.cuda.stream(s1 if it % 2 == 0 else s2):
            outs.append(dft.coset_lde_batch(x, 2, f.to_monty(5)).bit_reverse_rows())
    torch.cuda.synchronize()
    for o in outs:
        assert np.array_equal(host(o), exp)


def test_twiddle_cache_is_bounded(monkeypatch):
    """LRU eviction by bytes (P3GPU_TWIDDLE_CACHE_MB): many distinct coset shifts with a 1 MB cap stay correct."""
    from plonky3_b200.gpu import Gpu
    monkeypatch.setenv("P3GPU_TWIDDLE_CACHE_MB", "1")
    g = Gpu(0)
    f = KoalaBear
    dft = Radix2DitParallel(f, g)
    m = O.random_matrix(f.id, 1 << 14, 8, seed=71)
    x = dev(m)
    for k in range(2, 12):
        shift = f.to_monty(k)
        assert np.array_equal(host(dft.coset_dft_batch(x, shift)), O.coset_dft_batch(f.id, m, shift)), k
    for k in (2, 3):                                          # evicted entries are rebuilt
        assert np.array_equal(host(dft.coset_lde_batch(x, 1, f.to_monty(k)).bit_reverse_rows()), O.coset_lde_batch(f.id, m, 1, f.to_monty(k), bitrev_out=True))
    g.close()


@pytest.mark.parametrize("chunks", ["1", "3", "4", "7"])
def test_host_pointer_lde_is_pipelined_in_column_chunks(gpu, chunks, monkeypatch):
    """p3gpu_coset_lde_batch (host pointers): H2D || LDE || D2H over column chunks must equal the one-shot transform."""
    monkeypatch.setenv("P3GPU_E2E_CHUNKS", chunks)
    f = KoalaBear
    m = O.random_matrix(f.id, 1 << 16, 100, seed=81)                    # 26 MB: above the pipelining threshold
    exp = O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True)
    got = gpu.coset_lde_batch(f.id, m, 1, f.generator)
    assert np.array_equal(got, exp)
    pinned = torch.from_numpy(m.view(np.int32)).pin_memory()
    out = torch.empty((1 << 17, 100), dtype=torch.int32).pin_memory()
    _lib.check(gpu.L.p3gpu_coset_lde_batch(gpu.h, f.id, pinned.data_ptr(), 1 << 16, 100, 1, f.generator, out.data_ptr(), 1))
    assert np.array_equal(out.numpy().view(np.uint32), exp)
    got3 = gpu.coset_lde_batch(f.id, np.ascontiguousarray(m[:, :44]), 2, f.to_monty(11))           # ragged widths, blowup 4
    assert np.array_equal(got3, O.coset_lde_batch(f.id, np.ascontiguousarray(m[:, :44]), 2, f.to_monty(11), bitrev_out=True))


def test_pcs_commit_from_host_memory(gpu):
    """p3gpu_pcs_commit: host trace in, cap out, LDE + layers resident — equals the device-resident commit and the oracle."""
    f = KoalaBear
    mmcs, ohs = _mmcs_pair(f, "p2w24", gpu, cap_height=3)
    for log_h, w in [(10, 45), (15, 200)]:                                                         # serial path / chunked path
        m = O.random_matrix(f.id, 1 << log_h, w, seed=91)
        cap, lde, layers = gpu.pcs_commit_host(f.id, mmcs.hash_kind, m, 1, 3)
        elde = O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True)
        ol = O.merkle_tree(ohs, [elde])
        assert np.array_equal(host(lde), elde)
        assert np.array_equal(cap, O.merkle_cap(ol, 3))
        for a, b in zip(layers, ol):
            assert np.array_equal(host(a), b)


def test_batch_stark_fixture_main_commitment_on_gpu(gpu):
    """The reference's committed batch proof (batch-stark/tests/fixtures/batch_stark_two_adic_v1.postcard): its main commitment — ONE
    Merkle tree over the LDEs of both instance traces — reproduced with LDE and multi-matrix commit on the GPU."""
    from test_oracle import batch_fixture_main_cap
    gold = json.loads((GOLD / "batch_stark_two_adic_v1.json").read_text())
    pm = O.perm_from_rng(0, 16, O.SmallRng(777))
    perm = Poseidon2.new(BabyBear, 16, np.array(pm.rc_init)[:64].reshape(4, 16), np.array(pm.rc_term)[:64].reshape(4, 16),
                         np.array(pm.rc_int)[: pm.rounds_p], monty=True)
    mmcs = MerkleTreeMmcs.poseidon2(perm, None, 1, gpu)
    dft = Radix2DitParallel(BabyBear, gpu)
    for to in (lambda m: m, dev):                                      # host-pointer path and device-resident path
        cap = batch_fixture_main_cap(lambda m, bits, s: dft.coset_lde_batch(to(m), bits, s).bit_reverse_rows(), lambda mats: mmcs.commit(mats)[0])
        assert np.asarray(cap).tolist() == gold["main_cap"]
    default_poseidon2(BabyBear, 16).upload(gpu)                        # restore the default constants for the other tests


def test_cpp_host_mirror_pcs_commit_and_multi_opening(gpu, tmp_path):
    """include/p3gpu.hpp on the GPU: TwoAdicFriPcs::commit (host trace in, cap out, LDE + tree resident) and open_multi_batch with
    the pruned multiproof, from a C++ program (tests/cpp/pcs_commit_check.cpp), against the oracle; plus the small DFT/commit
    program of the link test."""
    import subprocess
    from plonky3_b200.merkle_tree import prune_paths
    root = pathlib.Path(__file__).resolve().parent.parent
    lib_dir = root / "plonky3_b200"

    def build(name):
        exe = tmp_path / name
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I", str(root / "include"), str(root / "tests" / "cpp" / f"{name}.cpp"), "-o", str(exe),
                        f"-L{lib_dir}", "-l:libp3gpu.so", f"-Wl,-rpath,{lib_dir}"], check=True)
        return exe
    r = subprocess.run([str(build("host_mirror_check"))], capture_output=True, text=True)
    assert r.returncode == 0 and "gpu ok" in r.stdout, r.stdout + r.stderr
    exe = build("pcs_commit_check")
    hs = O.keccak_hasher()
    for f, log_h, w, log_blowup, cap_height, idx in [(BabyBear, 6, 5, 1, 2, [5, 40, 41, 5, 127]), (KoalaBear, 10, 33, 2, 0, [0, 4095, 17, 18, 2048]),
                                                     (KoalaBear, 3, 1, 1, 3, [1, 15])]:
        r = subprocess.run([str(exe), str(f.id), str(_lib.HASH_KECCAK), str(log_h), str(w), str(log_blowup), str(cap_height), ",".join(map(str, idx))],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        lines = [l.split() for l in r.stdout.strip().splitlines()]
        words = lambda l: np.array([int(x, 16) for x in l[1:]], dtype=np.uint32)
        s, vals = 12345, []
        for _ in range((1 << log_h) * w):                         # the program's LCG
            s = (s * 6364136223846793005 + 1442695040888963407) & ((1 << 64) - 1)
            vals.append((s >> 33) % f.P)
        m = np.array(vals, dtype=np.uint32).reshape(1 << log_h, w)
        lde = O.coset_lde_batch(f.id, m, log_blowup, f.generator, bitrev_out=True)
        layers = O.merkle_tree(hs, [lde])
        eff = min(cap_height, len(layers) - 1)
        assert lines[0][0] == "cap" and np.array_equal(words(lines[0]).reshape(-1, 8), O.merkle_cap(layers, eff))
        rows = [words(l) for l in lines if l[0] == "row"]
        assert len(rows) == len(idx) and all(np.array_equal(r_, lde[i]) for r_, i in zip(rows, idx))
        paths = np.array([[layers[l][(i >> l) ^ 1] for l in range(len(layers) - 1 - eff)] for i in idx], dtype=np.uint32).reshape(len(idx), -1, 8)
        pruned = words([l for l in lines if l[0] == "pruned"][0]).reshape(-1, 8)
        assert np.array_equal(pruned, prune_paths(idx, paths))
