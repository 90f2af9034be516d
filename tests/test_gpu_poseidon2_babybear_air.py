"""The BabyBear instance of the Poseidon2 AIR's kernels on the GPU (csrc/air.cu, S-box degree 7 with one register): the trace
equals the restated generation bit for bit on a poisoned buffer; the quotient equals the constraint-DAG oracle on valid-trace and
random LDEs, is a polynomial of degree < 2N - 2 on a valid trace only, and equals the constraint-program kernel on the same DAG;
bad arguments are refused before any launch; two contexts keep their own field's constants; proofs under both configurations
have the stand-in device's bytes and pass the verifier; the example's own Poseidon2 configuration and the `-l 20` shape prove and
verify."""
import ctypes as C

import numpy as np
import pytest
import torch

import air_oracle as A
import poseidon2_babybear_air_oracle as BO
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200 import poseidon2_air as PA
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_keccak_air_cpu import corruption_sites
from test_poseidon2_babybear_air_cpu import COLS, NUM_QUERIES, POW_BITS, PROOF_CASES, WIDTH, _inputs, mock_prove

pytestmark = pytest.mark.gpu
f = BabyBear
POISON = -1                                                            # 0xffffffff: above p


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def _air(gpu, vector_len=PA.VECTOR_LEN, constants=None):
    return PA.VectorizedPoseidon2Air(f, constants or BO.example_constants(), gpu, vector_len=vector_len)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def _gen_poisoned(gpu, inputs):
    n = inputs.shape[0]
    _air(gpu)                                                          # sets BabyBear's constants on the context
    x = _dev(inputs)
    out = torch.full((n + 1, COLS), POISON, dtype=torch.int32, device="cuda")               # one guard row
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_p2air_generate_trace_dev(gpu.h, f.id, x.data_ptr(), n, out.data_ptr()))
    torch.cuda.synchronize()
    assert bool((out[-1] == POISON).all()), "write past the trace"
    return out[:-1]


@pytest.mark.parametrize("n", [8, 16, 40, 1 << 10, 1 << 17])
def test_trace_matches_the_oracle(gpu, n):
    inputs = _inputs(n, 50 + n)
    got = _gen_poisoned(gpu, inputs).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, BO.generate_perms(BO.example_constants(), inputs))


@pytest.mark.parametrize("vector_len", [1, 2, 8])
def test_trace_rows_wrapper(gpu, vector_len):
    inputs = _inputs(vector_len << 6, 9 + vector_len)
    w = _air(gpu, vector_len).generate_trace_rows(_dev(inputs))
    assert tuple(w.shape) == (64, vector_len * COLS)
    assert np.array_equal(w.cpu().numpy().view(np.uint32), BO.generate(BO.example_constants(), inputs, vector_len))


def _lde(gpu, trace_np, log_blowup):
    return gpu.coset_lde_batch(f.id, _dev(trace_np), log_blowup, f.generator, bitrev_rows=True)


def test_quotient_matches_the_dag_oracle(gpu):
    c = BO.example_constants()
    air = _air(gpu)
    nodes, cons = air.nodes, air.constraints
    rng = np.random.default_rng(7)
    for log_n in range(2, 11):
        valid = BO.generate(c, _inputs(8 << log_n, log_n))
        rand = rng.integers(0, f.P, (1 << log_n, WIDTH), dtype=np.uint32)
        for log_blowup in (1, 2):
            for kind, tr in (("valid", valid), ("random", rand)):
                lde = _lde(gpu, tr, log_blowup)
                alpha = rng.integers(0, f.P, 4, dtype=np.uint32)
                q = air.quotient_values(lde, log_n, alpha).cpu().numpy().view(np.uint32)
                exp = A.air_quotient(f.id, nodes, cons, lde.cpu().numpy().view(np.uint32), log_n + log_blowup, log_n, [], alpha)
                assert np.array_equal(q, exp), (log_n, log_blowup, kind)
                # coefficients over the coset: degree <= 3 (N - 1) - N = 2N - 3 exactly when the trace satisfies the AIR
                coeffs = O.coset_idft_batch(f.id, q, f.generator)
                assert (not np.any(coeffs[(2 << log_n) - 2:])) == (kind == "valid"), (log_n, log_blowup, kind)


def test_quotient_equals_the_restated_quotient(gpu):
    """The restatement of tests/poseidon2_babybear_air_oracle.py, written apart from the DAG, at 2^6 rows, vector lengths 1, 2, 8."""
    c = BO.example_constants()
    for vector_len in (1, 2, 8):
        air = _air(gpu, vector_len)
        tr = BO.generate(c, _inputs(vector_len << 6, 30 + vector_len), vector_len)
        lde = _lde(gpu, tr, 1)
        alpha = np.array([f.to_monty(v) for v in (2, 3, 5, 7)], dtype=np.uint32)
        q = air.quotient_values(lde, 6, alpha).cpu().numpy().view(np.uint32)
        assert np.array_equal(q, BO.quotient(c, lde.cpu().numpy().view(np.uint32), 6, alpha, vector_len)), vector_len


def test_quotient_equals_the_constraint_program(gpu):
    """A second, independent device check: at vector_len 1 (282 constraints) the constraint-program kernel (p3gpu_air_quotient_dev)
    on the same DAG at 2^10 rows gives the same quotient."""
    vector_len, log_n = 1, 10
    air = _air(gpu, vector_len)
    tr = BO.generate(BO.example_constants(), _inputs(vector_len << log_n, 9), vector_len)
    rand = np.random.default_rng(11).integers(0, f.P, tr.shape, dtype=np.uint32)
    prog = gpu.air_program_create(f.id, air.nodes, air.constraints, air.width(), 0)
    _, slots, n_cons = prog.info()
    assert n_cons == len(air.constraints) == 282 and slots <= 384
    for t in (tr, rand):
        lde = _lde(gpu, t, 1)
        alpha = np.array([f.to_monty(v) for v in (2, 3, 5, 7)], dtype=np.uint32)
        q = air.quotient_values(lde, log_n, alpha)
        p = gpu.air_quotient(prog, lde, log_n + 1, log_n, [], alpha)
        assert torch.equal(q, p), slots


def _consts_words(c):
    return [np.ascontiguousarray(np.asarray(a, dtype=np.uint32).ravel()) for a in
            (c.beginning_full_round_constants, c.partial_round_constants, c.ending_full_round_constants)]


def test_bad_arguments_are_refused_before_launch(gpu):
    L = gpu.L
    beg, part, end = _consts_words(BO.example_constants())
    ctx = C.c_void_p()
    _lib.check(L.p3gpu_ctx_create(0, C.byref(ctx)))
    try:
        x = torch.zeros((16, 16), dtype=torch.int32, device="cuda")
        t = torch.empty((16, COLS), dtype=torch.int32, device="cuda")
        lde = torch.zeros((5, COLS), dtype=torch.int32, device="cuda")          # a spare row for the offset LDE below
        q = torch.empty((4, 4), dtype=torch.int32, device="cuda")
        al = np.array([1, 2, 3, 4], dtype=np.uint32)
        torch.cuda.synchronize()                                       # the buffers exist before this context's stream reads them
        n0 = int(L.p3gpu_launch_count(ctx))
        gen, qd = L.p3gpu_p2air_generate_trace_dev, L.p3gpu_p2air_quotient_dev
        cols = L.p3gpu_p2air_generate_trace_cols_dev
        sh = L.p3gpu_p2air_quotient_sharded_dev
        # constants not set on this context
        assert gen(ctx, f.id, x.data_ptr(), 16, t.data_ptr()) == _lib.ESTATE
        assert qd(ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()) == _lib.ESTATE
        # set_constants: non-canonical words, rounds_p
        for i, (a, n) in enumerate(((beg, 64), (part, 13), (end, 64))):
            bad = [beg.copy(), part.copy(), end.copy()]
            bad[i][n - 1] = f.P
            assert L.p3gpu_p2air_set_constants(ctx, f.id, bad[0].ctypes.data, bad[1].ctypes.data, 13, bad[2].ctypes.data) == _lib.EINVAL, i
        long_part = np.zeros(40, dtype=np.uint32)
        for rp in (0, 33):
            assert L.p3gpu_p2air_set_constants(ctx, f.id, beg.ctypes.data, long_part.ctypes.data, rp, end.ctypes.data) == _lib.EINVAL, rp
        assert L.p3gpu_p2air_field_columns(f.id, 13) == 298 and L.p3gpu_p2air_field_columns(KoalaBear.id, 20) == 164
        assert L.p3gpu_p2air_field_columns(7, 13) == 0 and L.p3gpu_p2air_columns(20) == 164
        # constants set for the other field
        kc = O.air_from_rng(KoalaBear.id, O.SmallRng(1))
        kb, kp, ke = (np.array(kc.beg, dtype=np.uint32), np.array(kc.part, dtype=np.uint32)[:20], np.array(kc.end, dtype=np.uint32))
        _lib.check(L.p3gpu_p2air_set_constants(ctx, KoalaBear.id, kb.ctypes.data, kp.ctypes.data, 20, ke.ctypes.data))
        assert gen(ctx, f.id, x.data_ptr(), 16, t.data_ptr()) == _lib.ESTATE
        assert qd(ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()) == _lib.ESTATE
        _lib.check(L.p3gpu_p2air_set_constants(ctx, f.id, beg.ctypes.data, part.ctypes.data, 13, end.ctypes.data))
        assert gen(ctx, KoalaBear.id, x.data_ptr(), 16, t.data_ptr()) == _lib.ESTATE
        # an LDE that is not 8-byte aligned; a quotient that is not 16-byte aligned
        assert qd(ctx, f.id, 1, lde.data_ptr() + 4, 2, 1, al.ctypes.data, q.data_ptr()) == _lib.EINVAL
        assert qd(ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr() + 8) == _lib.EINVAL
        # the sharded entry points are KoalaBear-only
        cs = (C.c_size_t * 2)(0, COLS)
        assert cols(ctx, f.id, 1, x.data_ptr(), 16, 0, 4, t.data_ptr()) == _lib.EUNSUPPORTED
        assert sh(ctx, f.id, 1, None, cs, 2, 1, al.ctypes.data, q.data_ptr()) == _lib.EUNSUPPORTED
        assert int(L.p3gpu_launch_count(ctx)) == n0
        assert qd(ctx, f.id, 1, lde.data_ptr() + 8, 2, 1, al.ctypes.data, q.data_ptr()) == 0     # 8-byte aligned is enough
        _lib.check(L.p3gpu_ctx_sync(ctx))
    finally:
        L.p3gpu_ctx_destroy(ctx)


def test_contexts_keep_their_own_constants(gpu):
    """Two contexts with the two fields' constants: each generates its own field's trace."""
    from plonky3_b200.gpu import Gpu
    other = Gpu(0)
    try:
        bair = _air(other)
        kc = O.air_from_rng(KoalaBear.id, O.SmallRng(1))
        kair = PA.VectorizedPoseidon2Air(KoalaBear, PA.RoundConstants(np.array(kc.beg, np.uint32).reshape(4, 16),
                                                                      np.array(kc.part, np.uint32)[:20], np.array(kc.end, np.uint32).reshape(4, 16)), gpu)
        xb = _inputs(64, 1)
        xk = KoalaBear.to_monty_array(np.random.default_rng(2).integers(0, KoalaBear.P, (64, 16), dtype=np.uint64))
        tb = other.p2air_generate_trace(f.id, _dev(xb))
        tk = gpu.p2air_generate_trace(KoalaBear.id, _dev(xk))
        torch.cuda.synchronize()
        assert np.array_equal(tb.cpu().numpy().view(np.uint32), BO.generate(BO.example_constants(), xb))
        assert np.array_equal(tk.cpu().numpy().view(np.uint32), O.p2air_generate(O.air_from_rng(KoalaBear.id, O.SmallRng(1)), xk, 8))
        assert kair.width() == 1312 and bair.width() == WIDTH
    finally:
        other.close()


def _gpu_config(gpu, config_name):
    from test_poseidon1_air_cpu import p1_poseidon2_setup
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig
    if config_name == "keccak":
        m = MerkleTreeMmcs.keccak(f, cap_height=3, gpu=gpu)
        return KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters(1, 0, 3, NUM_QUERIES, 0, POW_BITS, m)))
    return p1_poseidon2_setup(f, gpu, NUM_QUERIES, POW_BITS, device_challenger=True)[0]


@pytest.mark.parametrize("config_name,rows", PROOF_CASES)
def test_gpu_proofs_have_the_stand_in_bytes(gpu, monkeypatch, config_name, rows):
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import prove, verify
    from plonky3_b200.verifier import VerificationError
    config = _gpu_config(gpu, config_name)
    air = _air(gpu)
    proof = prove(config, air, air.generate_trace_rows(_dev(_inputs(8 * rows, 7))))
    raw = proof.to_postcard()
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        _, mraw, vcfg = mock_prove(config_name, rows)
    assert raw == mraw
    vair = PA.VectorizedPoseidon2Air(f, BO.example_constants(), None)
    verify(vcfg, vair, raw)
    verify(config, air, raw)                                             # the product verifier with the device transcript
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, vair, bytes(bad))
        with pytest.raises(VerificationError):
            verify(config, air, bytes(bad))


def test_the_example_poseidon2_configuration(gpu):
    """prove_prime_field_31 -f baby-bear -o poseidon-2-permutations under its own configuration: the AIR's constants, then
    Poseidon2BabyBear<16> and <24> from new_from_rng_128, all from one SmallRng::seed_from_u64(1); the width-24 sponge as the
    Merkle leaf hash and the DuplexChallenger<24, 16>; 2^8 rows."""
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.poseidon2 import Poseidon2
    from plonky3_b200.uni_stark import StarkConfig, prove, verify
    from plonky3_b200.verifier import VerificationError
    rng = O.SmallRng(1)
    c = BO.constants_from_rng(rng)
    o16, o24 = O.perm_from_rng(f.id, 16, rng), O.perm_from_rng(f.id, 24, rng)
    assert (o16.rounds_p, o24.rounds_p) == (13, 21)
    mk = lambda pm: Poseidon2.new(f, pm.width, np.array(pm.rc_init)[: 4 * pm.width].reshape(4, pm.width),
                                  np.array(pm.rc_term)[: 4 * pm.width].reshape(4, pm.width), np.array(pm.rc_int)[: pm.rounds_p], monty=True)
    p24 = mk(o24)
    m = MerkleTreeMmcs.poseidon2(mk(o16), p24, cap_height=3, gpu=gpu)
    config = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters(1, 0, 3, 20, 0, 8, m)), p24, 16)
    air = _air(gpu, constants=c)
    inputs = O.SmallRng(1).field(f.id, 16 * (8 << 8)).reshape(-1, 16)
    raw = prove(config, air, air.generate_trace_rows(_dev(inputs))).to_postcard()
    verify(config, PA.VectorizedPoseidon2Air(f, c, None), raw)
    bad = bytearray(raw); bad[len(raw) // 2] ^= 1
    with pytest.raises(VerificationError):
        verify(config, PA.VectorizedPoseidon2Air(f, c, None), bytes(bad))


def test_full_shape_at_2_23_permutations(gpu):
    """`-f baby-bear -o poseidon-2-permutations -l 20`: 2^23 permutations (2^20 rows x 2384 columns, 10 GB, with a 20 GB LDE),
    the Keccak configuration with new_benchmark_high_arity and cap height 3, the reference's SmallRng(1) inputs."""
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig, prove, verify
    n = 1 << 23
    m = MerkleTreeMmcs.keccak(f, cap_height=3, gpu=gpu)
    config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)))
    air = _air(gpu)
    inputs = O.SmallRng(1).field(f.id, 16 * n).reshape(n, 16)
    trace = air.generate_trace_rows(_dev(inputs))
    assert tuple(trace.shape) == (1 << 20, WIDTH)
    c = BO.example_constants()
    for r in (0, (1 << 20) - 1):
        exp = BO.generate(c, inputs[8 * r: 8 * r + 8]).ravel()
        assert np.array_equal(trace[r].cpu().numpy().view(np.uint32), exp), r
    del inputs
    proof = prove(config, air, trace)
    del trace
    torch.cuda.empty_cache()
    verify(config, PA.VectorizedPoseidon2Air(f, c, None), proof.to_postcard())
