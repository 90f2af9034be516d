"""The Poseidon1 AIR (plonky3_b200.poseidon1_air) without a GPU: the fixture's known answers through a textbook Poseidon1, the
restated to_optimized against it, the restated generation's outputs, the constraint DAG (width, count, degree, vanishing on valid
traces, corruptions in every part of the row), the pinned random draw, KernelAir's guards, and proofs on the oracle-backed
stand-in device under both configurations, accepted by the product verifier and rejecting tampered bytes."""
import copy

import numpy as np
import pytest
import torch

import air_oracle as A
import keccak_air_oracle as KO
import mock_device as M
import poseidon1_air_oracle as PO
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200 import air as AIR
from plonky3_b200 import poseidon1_air as PA
from plonky3_b200.field import BabyBear, KoalaBear

FIELDS = [BabyBear, KoalaBear]
SHAPES = {BabyBear.id: (298, 2384, 2256), KoalaBear.id: (164, 1312, 1184)}     # columns, width, constraints


def _inputs(field, n, seed):
    """(n, 16) Montgomery inputs, with permutation 0 all zeros and permutation 1 all p - 1 (when there are such)."""
    x = np.random.default_rng(seed).integers(0, field.P, (n, 16), dtype=np.uint64)
    x[0] = 0
    if n > 1:
        x[1] = field.P - 1
    return field.to_monty_array(x)


class P1MockGpu(M.MockGpu):
    """The stand-in device with the Poseidon1 AIR's calls: the trace from the restated generation, the quotient from the
    constraint-DAG oracle (tests/air_oracle.py) on the AIR's DAG."""

    def p1air_set_constants(self, field, initial_full, terminal_full, mds_circ_col, first_round_constants, m_i, partial_rc,
                            sparse_first_row, v, rounds_p):
        f = BabyBear if field == BabyBear.id else KoalaBear
        c = lambda a: f.from_monty_array(M._n(a)).astype(np.int64)
        self.p1 = (f, PA.FullRoundConstants(c(initial_full), c(terminal_full), c(mds_circ_col)),
                   PA.PartialRoundConstants(c(first_round_constants), c(m_i).reshape(16, 16), c(sparse_first_row).reshape(rounds_p, 16),
                                            c(v).reshape(rounds_p, 16), c(partial_rc)))

    def p1air_generate_trace(self, field, inputs, vector_len=8):
        self._note("p1air_generate_trace")
        f, full, part = self.p1
        return M._t(PO.generate(f, full, part, inputs.contiguous().numpy().view(np.uint32), vector_len))

    def p1air_quotient(self, field, lde, log_trace_height, alpha, vector_len=8):
        self._note("p1air_quotient")
        f = self.p1[0]
        nodes, cons = PO.air_dag(f, vector_len)
        return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_trace_height + 1, log_trace_height, [], M._n(alpha)))


# ---------------------------------------------------------------- fixture, permutation, generation
@pytest.mark.parametrize("field", FIELDS)
def test_fixture_shape(field):
    fx = PO.fixture(field)
    rp = {BabyBear.id: 13, KoalaBear.id: 20}[field.id]
    assert (fx["rounds_f"], fx["rounds_p"], fx["sbox_degree"]) == (8, rp, field.SBOX_D)
    assert len(fx["round_constants"]) == 8 + rp and all(len(r) == 16 and all(0 <= v < field.P for v in r) for r in fx["round_constants"])
    # the first column of the circulant whose first row is mds.rs's [1, 1, 51, 1, 11, 17, 2, 1, 101, 63, 15, 2, 67, 22, 13, 3]
    row = [1, 1, 51, 1, 11, 17, 2, 1, 101, 63, 15, 2, 67, 22, 13, 3]
    assert PA.circulant(fx["mds_circ_col"], field.P)[0] == row


@pytest.mark.parametrize("field", FIELDS)
def test_textbook_reproduces_the_known_answer(field):
    fx = PO.fixture(field)
    out = PO.textbook(field, PO.raw_constants(field), np.array([fx["kat_input"]]))
    assert [int(v) for v in out[0]] == fx["kat_expected"]


@pytest.mark.parametrize("field", FIELDS)
def test_optimized_form_equals_the_textbook(field):
    fx = PO.fixture(field)
    full, part = PO.optimized(field)
    kat = PO.optimized_permutation(field, full, part, np.array([fx["kat_input"]]))
    assert [int(v) for v in kat[0]] == fx["kat_expected"]
    x = np.random.default_rng(100 + field.id).integers(0, field.P, (1000, 16), dtype=np.int64)
    assert np.array_equal(PO.optimized_permutation(field, full, part, x), PO.textbook(field, PO.raw_constants(field), x))


@pytest.mark.parametrize("field", FIELDS)
def test_optimized_constants_shapes(field):
    full, part = PO.optimized(field)
    rp = PO.fixture(field)["rounds_p"]
    assert np.asarray(full.initial).shape == (4, 16) and np.asarray(full.terminal).shape == (4, 16)
    assert np.asarray(part.m_i).shape == (16, 16) and part.rounds_p == rp
    assert np.asarray(part.sparse_first_row).shape == (rp, 16) and np.asarray(part.v).shape == (rp, 16)
    assert np.asarray(part.round_constants).shape == (rp - 1,) and not np.any(np.asarray(part.v)[:, 15])
    assert all(int(r[0]) == PO.fixture(field)["mds_circ_col"][0] for r in part.sparse_first_row)   # M[0][0]


@pytest.mark.parametrize("field", FIELDS)
def test_generation_outputs_are_the_permutation(field):
    full, part = PO.optimized(field)
    x = _inputs(field, 64, 3)
    t = PO.generate_perms(field, full, part, x)
    assert t.shape == (64, SHAPES[field.id][0]) and np.all(t < field.P)
    assert np.array_equal(t[:, :16], x)
    exp = PO.textbook(field, PO.raw_constants(field), field.from_monty_array(x).astype(np.int64))
    assert np.array_equal(PO.last_post(field, part, t), exp)
    v = PO.generate(field, full, part, x)
    assert v.shape == (8, SHAPES[field.id][1]) and np.array_equal(v.reshape(64, -1), t)
    with pytest.raises(AssertionError):
        PO.generate(field, full, part, x[:24])                      # 3 rows: not a power of two


@pytest.mark.parametrize("field", FIELDS)
def test_random_inputs_are_the_pinned_field_draw(field):
    a = PA.random_inputs(field, 6)
    assert a.shape == (6, 16) and a.dtype == np.uint32 and np.all(a < field.P)
    assert np.array_equal(a.ravel(), O.SmallRng(1).field(field.id, 96))
    assert np.array_equal(PA.random_inputs(field, 2), a[:2])


# ---------------------------------------------------------------- constraints
@pytest.mark.parametrize("field", FIELDS)
def test_width_count_and_degree_from_the_dag(field):
    air = PA.VectorizedPoseidon1Air(field, PO.optimized(field))
    cols, width, count = SHAPES[field.id]
    assert PA.columns(field, PO.fixture(field)["rounds_p"]) == cols
    degs = air.constraint_degrees()
    assert air.width() == width and len(degs) == count and max(degs) == 3 and air.max_constraint_degree() == 3
    assert air.num_public_values() == 0 and air.main_next_row_columns() == []
    assert not any(n[0] in (AIR.MAIN_NEXT, AIR.IS_FIRST_ROW, AIR.IS_LAST_ROW, AIR.IS_TRANSITION, AIR.PUBLIC) for n in air.nodes)
    one = PA.VectorizedPoseidon1Air(field, PO.optimized(field), vector_len=1)
    assert one.width() == cols and len(one.constraints) == count // 8


def _violated(field, tr):
    nodes, cons = PO.air_dag(field)
    return bool(np.any(KO.constraint_values(field.id, nodes, cons, tr)))


@pytest.mark.parametrize("field", FIELDS)
def test_constraints_vanish_on_valid_traces(field):
    full, part = PO.optimized(field)
    for n, seed in ((8, 1), (32, 2)):
        assert not _violated(field, PO.generate(field, full, part, _inputs(field, n, seed)))


@pytest.mark.parametrize("field", FIELDS)
def test_corruptions_are_detected(field):
    full, part = PO.optimized(field)
    reg, rp = PA.sbox_registers(field), part.rounds_p
    cols = SHAPES[field.id][0]
    fr = 16 * (reg + 1)
    base = PO.generate(field, full, part, _inputs(field, 16, 5))
    partial0 = 16 + 4 * fr
    sites = {"input": 3, "first full-round post": 16 + 16 * reg + 5, "third full-round post": 16 + 2 * fr + 16 * reg + 15,
             "partial post_sbox": partial0 + 7 * (reg + 1) + reg, "last partial post_sbox": partial0 + (rp - 1) * (reg + 1) + reg,
             "last post": cols - 1}
    if reg:
        sites.update({"full-round register": 16 + 2, "partial register": partial0 + 4 * (reg + 1), "ending register": partial0 + rp * 2 + fr + 9})
    add1 = lambda v: field.to_monty((field.from_monty(int(v)) + 1) % field.P)
    for name, c in sites.items():
        for v in (0, 3, 7):                                          # permutation 0, 3 and the last one of the row
            for row in (0, 1):
                tr = base.copy()
                tr[row, v * cols + c] = add1(tr[row, v * cols + c])
                assert _violated(field, tr), (name, v, row)


# ---------------------------------------------------------------- KernelAir's guards
class RecordingGpu:
    """Records every call; answers a quotient call with a token and computes nothing."""
    device = None

    def __init__(self):
        self.calls = []

    def p1air_set_constants(self, *args): self.calls.append(("p1air_set_constants", args))

    def p1air_quotient(self, *args):
        self.calls.append(("p1air_quotient", args))
        return ("quotient", args)


def test_kernel_air_guards_refuse_before_the_device():
    rg = RecordingGpu()
    air = PA.VectorizedPoseidon1Air(KoalaBear, PO.optimized(KoalaBear), rg, vector_len=4)
    lde, al = np.zeros((16, air.width()), dtype=np.uint32), np.array([1, 2, 3, 4], dtype=np.uint32)
    n0 = len(rg.calls)
    with pytest.raises(ValueError, match="Poseidon1 AIR has none"):
        air.quotient_values(lde, 3, al, public_values=[1])
    with pytest.raises(ValueError, match="Poseidon1 AIR has no preprocessed"):
        air.quotient_values(lde, 3, al, preprocessed_on_quotient_domain=lde)
    assert len(rg.calls) == n0
    air.gpu = None
    with pytest.raises(_lib.P3GpuError, match="needs a GPU context"):
        air.quotient_values(lde, 3, al)
    with pytest.raises(_lib.P3GpuError, match="needs a GPU context"):
        air.generate_trace_rows(torch.zeros((4, 16), dtype=torch.int32))
    air.gpu = rg
    assert air.quotient_values(lde, 3, al)[0] == "quotient"
    name, args = rg.calls[-1]
    assert name == "p1air_quotient" and args[0] == KoalaBear.id and args[1] is lde and args[2] == 3 and args[3] is al and args[4] == 4
    # the constants reach the device in Montgomery form, as to_optimized's canonical values
    full, part = PO.optimized(KoalaBear)
    consts = [c for c in rg.calls if c[0] == "p1air_set_constants"][-1][1]
    assert consts[0] == KoalaBear.id and consts[-1] == 20
    assert np.array_equal(KoalaBear.from_monty_array(consts[5]), np.asarray(part.m_i, dtype=np.uint32))


# ---------------------------------------------------------------- proofs on the stand-in device
PROOF_CASES = [(f, c, rows) for f in FIELDS for c in ("poseidon2", "keccak") for rows in (1 << 3, 1 << 6)]
NUM_QUERIES, POW_BITS = 6, 3


def p1_poseidon2_setup(field, gpu, num_queries, pow_bits, device_challenger=False):
    """The Poseidon2 configuration of the Poseidon1 objective: BabyBear as tests/test_keccak_air_cpu.poseidon2_setup; KoalaBear's
    Merkle / transcript Poseidon2-16 and -24 are the FIRST draws of SmallRng::seed_from_u64(1) (no draw is spent on the AIR, whose
    constants are fixed)."""
    from types import SimpleNamespace
    import p2_prove_replay as R
    from test_keccak_air_cpu import poseidon2_setup
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.poseidon2 import Poseidon2
    if field is BabyBear:
        return poseidon2_setup(field, gpu, num_queries, pow_bits, device_challenger)
    rng = O.SmallRng(1)
    o16, o24 = O.perm_from_rng(field.id, 16, rng), O.perm_from_rng(field.id, 24, rng)
    mk = lambda pm: Poseidon2.new(field, pm.width, np.array(pm.rc_init)[: 4 * pm.width].reshape(4, pm.width),
                                  np.array(pm.rc_term)[: 4 * pm.width].reshape(4, pm.width), np.array(pm.rc_int)[: pm.rounds_p], monty=True)
    p24 = mk(o24)
    mmcs = MerkleTreeMmcs.poseidon2(mk(o16), p24, cap_height=3, gpu=gpu)
    cfg = R.verifier_config(o16, o24)
    cfg.update(log_blowup=1, log_final_poly_len=0, max_log_arity=3, num_queries=num_queries, commit_pow_bits=0, query_pow_bits=pow_bits)
    pcs = TwoAdicFriPcs(Radix2DitParallel(field, gpu), mmcs, FriParameters(1, 0, 3, num_queries, 0, pow_bits, mmcs))
    if device_challenger:
        from plonky3_b200.uni_stark import StarkConfig
        return StarkConfig(pcs, p24, 16), cfg
    return SimpleNamespace(pcs=pcs, initialise_challenger=lambda: M.MockChallenger(o24)), cfg


def mock_prove(field, config_name, rows):
    """(proof, raw bytes, product verifier config) of the Poseidon1 AIR over `rows` rows (8 rows per permutation group) on the
    stand-in device."""
    import keccak_transcript as K
    import stark_verify as V
    from plonky3_b200.uni_stark import prove
    mock = P1MockGpu()
    if config_name == "keccak":
        config = K.keccak_mock_config(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = K.verifier_config(field, NUM_QUERIES, POW_BITS)
    else:
        config, cfg = p1_poseidon2_setup(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = V.product_config(field, cfg)
    air = PA.VectorizedPoseidon1Air(field, PO.optimized(field), mock)
    trace = air.generate_trace_rows(torch.from_numpy(_inputs(field, 8 * rows, 7).view(np.int32)))
    proof = prove(config, air, trace)
    assert "p1air_quotient" in mock.calls
    return proof, proof.to_postcard(), vcfg


@pytest.mark.parametrize("field,config_name,rows", PROOF_CASES)
def test_proofs_on_the_stand_in_device(monkeypatch, field, config_name, rows):
    from test_keccak_air_cpu import corruption_sites
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import verify
    from plonky3_b200.verifier import VerificationError
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    proof, raw, vcfg = mock_prove(field, config_name, rows)
    assert proof.degree_bits == rows.bit_length() - 1 and len(proof.quotient_chunks) == 2
    assert proof.trace_next is None and len(proof.trace_local) == SHAPES[field.id][1]
    verifier_air = PA.VectorizedPoseidon1Air(field, PO.optimized(field))        # verifier-only: no device
    verify(vcfg, verifier_air, raw)
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, verifier_air, bytes(bad))
    # a proof whose opened row breaks a constraint is rejected at the out-of-domain check
    bad = copy.deepcopy(proof)
    bad.trace_local = np.array(bad.trace_local, dtype=np.uint32)
    col = 7 * SHAPES[field.id][0] + 100
    bad.trace_local[col, 0] = (int(bad.trace_local[col, 0]) + 1) % field.P
    with pytest.raises(VerificationError):
        verify(vcfg, verifier_air, bad.to_postcard())
