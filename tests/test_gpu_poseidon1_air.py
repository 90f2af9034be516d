"""The Poseidon1 AIR's kernels on the GPU (csrc/poseidon1_air.cu): the trace equals the restated generation bit for bit on a
poisoned buffer; the quotient equals the constraint-DAG oracle on valid-trace and random LDEs, is a polynomial of degree < 2N - 2
on a valid trace only, and equals the constraint-program kernel on the same DAG; bad arguments are refused before any launch;
proofs under both configurations have the stand-in device's bytes and pass the verifier; the `-l 20` shape proves and verifies."""
import numpy as np
import pytest
import torch

import air_oracle as A
import poseidon1_air_oracle as PO
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200 import poseidon1_air as PA
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_keccak_air_cpu import corruption_sites
from test_poseidon1_air_cpu import FIELDS, NUM_QUERIES, POW_BITS, PROOF_CASES, SHAPES, _inputs, mock_prove, p1_poseidon2_setup

pytestmark = pytest.mark.gpu
POISON = -1                                                            # 0xffffffff: above p in both fields


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def _air(gpu, field, vector_len=PA.VECTOR_LEN):
    return PA.VectorizedPoseidon1Air(field, PO.optimized(field), gpu, vector_len=vector_len)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def _gen_poisoned(gpu, field, inputs):
    n, cols = inputs.shape[0], SHAPES[field.id][0]
    _air(gpu, field)                                                   # sets this field's constants on the context
    x = _dev(inputs)
    out = torch.full((n + 1, cols), POISON, dtype=torch.int32, device="cuda")           # one guard row
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_p1air_generate_trace_dev(gpu.h, field.id, x.data_ptr(), n, out.data_ptr()))
    torch.cuda.synchronize()
    assert bool((out[-1] == POISON).all()), "write past the trace"
    return out[:-1]


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [8, 16, 40, 1 << 10, 1 << 17])
def test_trace_matches_the_oracle(gpu, field, n):
    full, part = PO.optimized(field)
    inputs = _inputs(field, n, 50 + n)
    got = _gen_poisoned(gpu, field, inputs).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, PO.generate_perms(field, full, part, inputs))
    if n == 1 << 10:                                                   # the generate_trace_rows wrapper writes the same
        w = _air(gpu, field).generate_trace_rows(_dev(inputs))
        assert tuple(w.shape) == (n // 8, SHAPES[field.id][1])
        assert np.array_equal(w.cpu().numpy().view(np.uint32).reshape(n, -1), got)


def _lde(gpu, field, trace_np, log_blowup):
    return gpu.coset_lde_batch(field.id, _dev(trace_np), log_blowup, field.generator, bitrev_rows=True)


@pytest.mark.parametrize("field", FIELDS)
def test_quotient_matches_the_dag_oracle(gpu, field):
    full, part = PO.optimized(field)
    air = _air(gpu, field)
    nodes, cons = PO.air_dag(field)
    rng = np.random.default_rng(7 + field.id)
    for log_n in range(2, 11):
        valid = PO.generate(field, full, part, _inputs(field, 8 << log_n, log_n))
        rand = rng.integers(0, field.P, (1 << log_n, air.width()), dtype=np.uint32)
        for log_blowup in (1, 2):
            for kind, tr in (("valid", valid), ("random", rand)):
                lde = _lde(gpu, field, tr, log_blowup)
                alpha = rng.integers(0, field.P, 4, dtype=np.uint32)
                q = air.quotient_values(lde, log_n, alpha).cpu().numpy().view(np.uint32)
                exp = A.air_quotient(field.id, nodes, cons, lde.cpu().numpy().view(np.uint32), log_n + 1, log_n, [], alpha)
                assert np.array_equal(q, exp), (log_n, log_blowup, kind)
                if log_blowup == 1:
                    # coefficients over the coset: degree <= 3 (N - 1) - N = 2N - 3 exactly when the trace satisfies the AIR
                    coeffs = O.coset_idft_batch(field.id, q, field.generator)
                    assert (not np.any(coeffs[(2 << log_n) - 2:])) == (kind == "valid"), (log_n, kind)


@pytest.mark.parametrize("field", FIELDS)
def test_quotient_equals_the_constraint_program(gpu, field):
    """A second, independent device check: at vector_len 1 (282 and 148 constraints, about 100 slots) the constraint-program kernel
    (p3gpu_air_quotient_dev) on the same DAG at 2^10 rows gives the same quotient."""
    full, part = PO.optimized(field)
    vector_len = 1
    air = _air(gpu, field, vector_len)
    log_n = 10
    tr = PO.generate(field, full, part, _inputs(field, vector_len << log_n, 9), vector_len)
    rand = np.random.default_rng(11).integers(0, field.P, tr.shape, dtype=np.uint32)
    prog = gpu.air_program_create(field.id, air.nodes, air.constraints, air.width(), 0)
    _, slots, n_cons = prog.info()
    assert n_cons == len(air.constraints) and slots <= 384
    for t in (tr, rand):
        lde = _lde(gpu, field, t, 1)
        alpha = np.array([field.to_monty(v) for v in (2, 3, 5, 7)], dtype=np.uint32)
        q = air.quotient_values(lde, log_n, alpha)
        p = gpu.air_quotient(prog, lde, log_n + 1, log_n, [], alpha)
        assert torch.equal(q, p), (field.name, vector_len, slots)


def test_vector_len_8_is_past_the_constraint_program_limits(gpu):
    """At vector_len 8 the constraint-program path cannot check this AIR: KoalaBear's 1,184 constraints fit its 2,048, but the eight
    permutations share every round constant and matrix entry, whose values stay live across the whole program: more than its 384
    slots.  BabyBear's 2,256 constraints are past 2,048."""
    for field, what in ((KoalaBear, "slots"), (BabyBear, "constraints")):
        air = _air(None, field)
        with pytest.raises(_lib.P3GpuError, match=what) as e:
            gpu.air_program_create(field.id, air.nodes, air.constraints, air.width(), 0)
        assert e.value.code == _lib.EUNSUPPORTED


def test_bad_arguments_are_refused_before_launch(gpu):
    f = KoalaBear
    L = gpu.L
    full, part = PO.optimized(f)
    mo = lambda a: f.to_monty_array(np.asarray(a, dtype=np.int64) % f.P).ravel()
    args = [mo(full.initial), mo(full.terminal), mo(full.mds_circ_col), mo(part.first_round_constants), mo(part.m_i),
            mo(part.round_constants), mo(part.sparse_first_row), mo(part.v)]
    ptrs = [a.ctypes.data for a in args]
    import ctypes as C
    ctx = C.c_void_p()
    _lib.check(L.p3gpu_ctx_create(0, C.byref(ctx)))
    try:
        x = torch.zeros((16, 16), dtype=torch.int32, device="cuda")
        t = torch.empty((16, 164), dtype=torch.int32, device="cuda")
        q = torch.empty((4, 4), dtype=torch.int32, device="cuda")
        al = np.array([1, 2, 3, 4], dtype=np.uint32)
        torch.cuda.synchronize()                                       # the buffers exist before this context's stream reads them
        # constants not set on this context
        assert L.p3gpu_p1air_generate_trace_dev(ctx, f.id, x.data_ptr(), 16, t.data_ptr()) == _lib.ESTATE
        assert L.p3gpu_p1air_quotient_dev(ctx, f.id, 8, t.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()) == _lib.ESTATE
        # set_constants: nulls, non-canonical words, rounds_p, field
        assert L.p3gpu_p1air_set_constants(ctx, f.id, None, *ptrs[1:], 20) == _lib.EINVAL
        assert L.p3gpu_p1air_set_constants(ctx, f.id, *ptrs[:7], None, 20) == _lib.EINVAL
        for i in range(8):
            bad = [a.copy() for a in args]
            bad[i][0] = f.P
            assert L.p3gpu_p1air_set_constants(ctx, f.id, *[a.ctypes.data for a in bad], 20) == _lib.EINVAL, i
        big = [a.copy() for a in args]
        big[2][1] = f.to_monty(1 << 12)                                # a circulant entry the kernels cannot take
        assert L.p3gpu_p1air_set_constants(ctx, f.id, *[a.ctypes.data for a in big], 20) == _lib.EINVAL
        for rp in (0, 18, 36, -4):
            assert L.p3gpu_p1air_set_constants(ctx, f.id, *ptrs, rp) == _lib.EINVAL, rp
        assert L.p3gpu_p1air_set_constants(ctx, 7, *ptrs, 20) == _lib.EUNSUPPORTED
        assert L.p3gpu_p1air_columns(7, 20) == 0 and L.p3gpu_p1air_columns(f.id, 20) == 164 and L.p3gpu_p1air_columns(BabyBear.id, 13) == 298
        _lib.check(L.p3gpu_p1air_set_constants(ctx, f.id, *ptrs, 20))
        # constants set for the other field
        assert L.p3gpu_p1air_generate_trace_dev(ctx, BabyBear.id, x.data_ptr(), 16, t.data_ptr()) == _lib.ESTATE
        assert L.p3gpu_p1air_quotient_dev(ctx, BabyBear.id, 8, t.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()) == _lib.ESTATE
        n0 = int(L.p3gpu_launch_count(ctx))
        gen = L.p3gpu_p1air_generate_trace_dev
        assert gen(ctx, f.id, None, 16, t.data_ptr()) == _lib.EINVAL
        assert gen(ctx, f.id, x.data_ptr(), 16, None) == _lib.EINVAL
        assert gen(ctx, f.id, x.data_ptr() + 4, 16, t.data_ptr()) == _lib.EINVAL                  # inputs not 16-byte aligned
        assert gen(ctx, f.id, x.data_ptr(), 16, t.data_ptr() + 2) == _lib.EINVAL
        assert gen(ctx, f.id, x.data_ptr(), 0, t.data_ptr()) == _lib.EINVAL                       # no permutations
        assert gen(ctx, 7, x.data_ptr(), 16, t.data_ptr()) == _lib.EUNSUPPORTED
        # quotient over a 2-row trace of vector_len 1 (an LDE of 4 rows x 164)
        lde = torch.zeros((4, 164), dtype=torch.int32, device="cuda")
        qd = L.p3gpu_p1air_quotient_dev
        ok = (ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr())
        cases = [
            ((ctx, f.id, 1, None, 2, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),
            ((ctx, f.id, 1, lde.data_ptr(), 2, 1, None, q.data_ptr()), _lib.EINVAL),
            ((ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, None), _lib.EINVAL),
            ((ctx, f.id, 3, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),      # not a power of two
            ((ctx, f.id, 64, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),     # above 32
            ((ctx, f.id, 0, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),
            ((ctx, f.id, 1, lde.data_ptr() + 8, 2, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),  # KoalaBear: 16-byte loads
            ((ctx, f.id, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr() + 1), _lib.EINVAL),
            ((ctx, f.id, 1, lde.data_ptr(), 2, 2, al.ctypes.data, q.data_ptr()), _lib.EINVAL),      # log_trace_height + 1 > log_lde
            ((ctx, f.id, 1, lde.data_ptr(), 30, 1, al.ctypes.data, q.data_ptr()), _lib.EINVAL),     # above the two-adicity
            ((ctx, f.id, 1, lde.data_ptr(), 2, 1, np.array([f.P, 0, 0, 0], np.uint32).ctypes.data, q.data_ptr()), _lib.EINVAL),
            ((ctx, 7, 1, lde.data_ptr(), 2, 1, al.ctypes.data, q.data_ptr()), _lib.EUNSUPPORTED),
        ]
        for a, code in cases:
            assert qd(*a) == code, a
        assert int(L.p3gpu_launch_count(ctx)) == n0
        assert qd(*ok) == 0                                            # and the valid call runs
        _lib.check(L.p3gpu_ctx_sync(ctx))
    finally:
        L.p3gpu_ctx_destroy(ctx)


def test_contexts_keep_their_own_constants(gpu):
    """Two contexts with the two fields' constants: each generates its own field's trace."""
    from plonky3_b200.gpu import Gpu
    other = Gpu(0)
    try:
        _air(other, BabyBear)
        _air(gpu, KoalaBear)
        xb, xk = _inputs(BabyBear, 64, 1), _inputs(KoalaBear, 64, 2)
        tb = _air(other, BabyBear).generate_trace_rows(_dev(xb))
        tk = gpu.p1air_generate_trace(KoalaBear.id, _dev(xk))
        torch.cuda.synchronize()
        assert np.array_equal(tb.cpu().numpy().view(np.uint32).reshape(64, -1), PO.generate_perms(BabyBear, *PO.optimized(BabyBear), xb))
        assert np.array_equal(tk.cpu().numpy().view(np.uint32).reshape(64, -1), PO.generate_perms(KoalaBear, *PO.optimized(KoalaBear), xk))
    finally:
        other.close()


def _gpu_config(gpu, field, config_name):
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig
    if config_name == "keccak":
        m = MerkleTreeMmcs.keccak(field, cap_height=3, gpu=gpu)
        return KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m, FriParameters(1, 0, 3, NUM_QUERIES, 0, POW_BITS, m)))
    return p1_poseidon2_setup(field, gpu, NUM_QUERIES, POW_BITS, device_challenger=True)[0]


@pytest.mark.parametrize("field,config_name,rows", PROOF_CASES)
def test_gpu_proofs_have_the_stand_in_bytes(gpu, monkeypatch, field, config_name, rows):
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import prove, verify
    from plonky3_b200.verifier import VerificationError
    config = _gpu_config(gpu, field, config_name)
    air = _air(gpu, field)
    proof = prove(config, air, air.generate_trace_rows(_dev(_inputs(field, 8 * rows, 7))))
    raw = proof.to_postcard()
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        _, mraw, vcfg = mock_prove(field, config_name, rows)
    assert raw == mraw
    vair = PA.VectorizedPoseidon1Air(field, PO.optimized(field))
    verify(vcfg, vair, raw)
    verify(config, air, raw)                                             # the product verifier with the device transcript
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, vair, bytes(bad))


@pytest.mark.parametrize("field", FIELDS)
def test_full_shape_at_2_23_permutations(gpu, field):
    """`-o poseidon-1-permutations -l 20`: 2^23 permutations (2^20 rows; KoalaBear 1312 columns, 5.5 GB, BabyBear 2384, 10 GB), the
    Keccak configuration with new_benchmark_high_arity and cap height 3, the reference's SmallRng(1) inputs."""
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig, prove, verify
    n = 1 << 23
    m = MerkleTreeMmcs.keccak(field, cap_height=3, gpu=gpu)
    config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m, FriParameters.new_benchmark_high_arity(m)))
    air = _air(gpu, field)
    inputs = O.SmallRng(1).field(field.id, 16 * n).reshape(n, 16)      # PA.random_inputs(field, n), drawn by the C oracle
    trace = air.generate_trace_rows(_dev(inputs))
    assert tuple(trace.shape) == (1 << 20, SHAPES[field.id][1])
    full, part = PO.optimized(field)
    for r in (0, (1 << 20) - 1):
        exp = PO.generate(field, full, part, inputs[8 * r: 8 * r + 8]).ravel()
        assert np.array_equal(trace[r].cpu().numpy().view(np.uint32), exp), r
    del inputs
    proof = prove(config, air, trace)
    del trace
    torch.cuda.empty_cache()
    verify(config, PA.VectorizedPoseidon1Air(field, PO.optimized(field)), proof.to_postcard())
