"""The BabyBear Poseidon2 AIR (plonky3_b200.poseidon2_air, S-box degree 7 with one register) without a GPU: the DAG's shape, the
restated generation against the C oracle's permutation (pinned by the reference's known answers) and against x3 = x^3, the DAG's
constraint values against the independent restatement (tests/poseidon2_babybear_air_oracle.py) and on corrupted traces, the two
quotient oracles against each other, the sharded prove's refusal, and proofs on the oracle-backed stand-in device under both
configurations, accepted by the product verifier and rejecting tampered bytes."""
import json
import pathlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import air_oracle as A
import keccak_air_oracle as KO
import mock_device as M
import poseidon2_babybear_air_oracle as BO
from oracle import p3_oracle as O
from plonky3_b200 import air as AIR
from plonky3_b200 import poseidon2_air as PA
from plonky3_b200.field import BabyBear

f = BabyBear
COLS, WIDTH, CONSTRAINTS = 298, 2384, 2256
GOLD = pathlib.Path(__file__).resolve().parent / "golden"


def _inputs(n, seed):
    """(n, 16) Montgomery inputs, with permutation 0 all zeros and permutation 1 all p - 1 (when there are such)."""
    x = np.random.default_rng(seed).integers(0, f.P, (n, 16), dtype=np.uint64)
    x[0] = 0
    if n > 1:
        x[1] = f.P - 1
    return f.to_monty_array(x)


class BabyBearP2MockGpu(M.MockGpu):
    """The stand-in device with the BabyBear Poseidon2 AIR's calls answered by the restatement: the trace from its generation, the
    quotient from its constraint values (not from the AIR's DAG)."""

    def p2air_set_constants(self, field, beginning_full, partial, ending_full):
        assert field == f.id
        self.p2 = PA.RoundConstants(M._n(beginning_full).reshape(4, 16), M._n(partial).ravel(), M._n(ending_full).reshape(4, 16))

    def p2air_generate_trace(self, field, inputs, vector_len=8):
        self._note("p2air_generate_trace")
        return M._t(BO.generate(self.p2, M._n(inputs), vector_len))

    def p2air_quotient(self, field, lde, log_trace_height, alpha, vector_len=8):
        self._note("p2air_quotient")
        return M._t(BO.quotient(self.p2, M._n(lde), log_trace_height, M._n(alpha), vector_len))


# ---------------------------------------------------------------- the DAG's shape
def test_width_count_and_degree_from_the_dag():
    from plonky3_b200.uni_stark import get_log_num_quotient_chunks
    c = BO.example_constants()
    air = PA.VectorizedPoseidon2Air(f, c, None)
    assert PA.sbox_registers(f) == 1 and PA.columns(f, 13) == COLS == BO.COLS
    degs = air.constraint_degrees()
    assert air.width() == WIDTH and len(degs) == CONSTRAINTS and max(degs) == 3 and air.max_constraint_degree() == 3
    assert air.num_public_values() == 0 and air.main_next_row_columns() == []
    assert not any(n[0] in (AIR.MAIN_NEXT, AIR.IS_FIRST_ROW, AIR.IS_LAST_ROW, AIR.IS_TRANSITION, AIR.PUBLIC) for n in air.nodes)
    assert 1 << get_log_num_quotient_chunks(air) == 2
    one = PA.VectorizedPoseidon2Air(f, c, None, vector_len=1)
    assert one.width() == COLS and len(one.constraints) == CONSTRAINTS // 8 == BO.CONSTRAINTS


def test_constants_are_the_example_draws():
    """RoundConstants::from_rng on SmallRng(1): 64 beginning, 13 partial, 64 ending words, in that order."""
    c = BO.example_constants()
    draw = O.SmallRng(1).field(f.id, 64 + 13 + 64)
    assert np.array_equal(np.asarray(c.beginning_full_round_constants).ravel(), draw[:64])
    assert np.array_equal(np.asarray(c.partial_round_constants), draw[64:77])
    assert np.array_equal(np.asarray(c.ending_full_round_constants).ravel(), draw[77:])


# ---------------------------------------------------------------- generation
def test_the_oracle_permutation_is_pinned_by_the_known_answer():
    kat = json.loads((GOLD / "poseidon2_kat.json").read_text())["baby_bear_16"]
    out = O.poseidon2_permute(O.default_perm(f.id, 16), O.to_monty_arr(f.id, kat["input"]))
    assert O.from_monty_arr(f.id, out).tolist() == kat["expected"]


def test_generation_outputs_are_the_permutation():
    c = BO.example_constants()
    x = _inputs(64, 3)
    t = BO.generate_perms(c, x)
    assert t.shape == (64, COLS) and np.all(t < f.P) and np.array_equal(t[:, :16], x)
    perm = BO.permutation(c)
    for i in range(64):
        assert np.array_equal(t[i, -16:], O.poseidon2_permute(perm, x[i])), i
    v = BO.generate(c, x)
    assert v.shape == (8, WIDTH) and np.array_equal(v.reshape(64, -1), t)


def test_every_register_is_the_cube_of_its_sbox_input():
    """Replays the permutation from the trace's own committed columns: every register equals (state + rc)^3."""
    c = BO.example_constants()
    beg, part, end = BO._canon(c)
    t = f.from_monty_array(BO.generate_perms(c, _inputs(32, 4))).astype(np.int64)
    p = f.P
    cube = lambda v: v * v % p * v % p
    s = BO._mds_light(t[:, :16])
    k = 16
    for rc in beg:
        assert np.array_equal(t[:, k:k + 16], cube((s + rc) % p)), k
        s = t[:, k + 16:k + 32]; k += 32
    for r in range(13):
        assert np.array_equal(t[:, k], cube((s[:, 0] + part[r]) % p)), k
        s = s.copy(); s[:, 0] = t[:, k + 1]
        s = BO._internal(s); k += 2
    for rc in end:
        assert np.array_equal(t[:, k:k + 16], cube((s + rc) % p)), k
        s = t[:, k + 16:k + 32]; k += 32
    assert k == COLS


# ---------------------------------------------------------------- constraints
def _dag(vector_len=8):
    air = PA.VectorizedPoseidon2Air(f, BO.example_constants(), None, vector_len=vector_len)
    return air.nodes, air.constraints


def test_dag_constraint_values_equal_the_restatement():
    """Value, order and sign of every constraint: the DAG's on random rows equal the restatement's."""
    nodes, cons = _dag()
    tr = np.random.default_rng(5).integers(0, f.P, (4, WIDTH), dtype=np.uint32)
    got = KO.constraint_values(f.id, nodes, cons, tr)
    assert np.array_equal(got.T, BO.constraint_values(BO.example_constants(), tr))


def test_constraints_vanish_on_valid_traces():
    nodes, cons = _dag()
    c = BO.example_constants()
    for n, seed in ((8, 1), (32, 2)):
        tr = BO.generate(c, _inputs(n, seed))
        assert not np.any(KO.constraint_values(f.id, nodes, cons, tr))
        assert not np.any(BO.constraint_values(c, tr))


def test_one_flipped_word_in_each_column_class_is_detected():
    nodes, cons = _dag()
    base = BO.generate(BO.example_constants(), _inputs(16, 5))
    partial0 = 16 + 4 * 32
    sites = {"input": 3, "full-round register": 16 + 2, "full-round post": 16 + 16 + 5, "third full-round post": 16 + 2 * 32 + 16 + 15,
             "partial register": partial0 + 4 * 2, "partial post_sbox": partial0 + 7 * 2 + 1, "last post_sbox": partial0 + 12 * 2 + 1,
             "ending register": partial0 + 26 + 32 + 9, "last post": COLS - 1}
    add1 = lambda v: f.to_monty((f.from_monty(int(v)) + 1) % f.P)
    for name, col in sites.items():
        for v in (0, 3, 7):
            for row in (0, 1):
                tr = base.copy()
                tr[row, v * COLS + col] = add1(tr[row, v * COLS + col])
                assert np.any(KO.constraint_values(f.id, nodes, cons, tr)), (name, v, row)


# ---------------------------------------------------------------- the two quotient oracles
@pytest.mark.parametrize("log_n,log_blowup,vector_len", [(2, 1, 8), (3, 2, 8), (4, 1, 1), (3, 1, 2)])
def test_dag_quotient_equals_the_restated_quotient(log_n, log_blowup, vector_len):
    c = BO.example_constants()
    nodes, cons = _dag(vector_len)
    rng = np.random.default_rng(40 + log_n)
    valid = BO.generate(c, _inputs(vector_len << log_n, log_n), vector_len)
    rand = rng.integers(0, f.P, valid.shape, dtype=np.uint32)
    for tr in (valid, rand):
        lde = O.coset_lde_batch(f.id, tr, log_blowup, f.generator, bitrev_out=True)
        alpha = rng.integers(0, f.P, 4, dtype=np.uint32)
        exp = A.air_quotient(f.id, nodes, cons, lde, log_n + log_blowup, log_n, [], alpha)
        assert np.array_equal(BO.quotient(c, lde, log_n, alpha, vector_len), exp)


# ---------------------------------------------------------------- the sharded prove is KoalaBear-only
def test_prove_sharded_refuses_babybear_before_the_group():
    from plonky3_b200 import distributed as D

    class Untouchable:
        """A PeerGroup whose every attribute but `gpu` fails: any collective or allocation would reach one."""
        def __init__(self, gpu): object.__setattr__(self, "_gpu", gpu)
        def __getattr__(self, name):
            if name == "gpu":
                return self._gpu
            raise AssertionError(f"prove_sharded reached the group's {name}")
    dev = object()
    config = SimpleNamespace(pcs=SimpleNamespace(dft=SimpleNamespace(gpu=dev)))
    air = PA.VectorizedPoseidon2Air(f, BO.example_constants(), None)
    with pytest.raises(ValueError, match="KoalaBear only"):
        D.prove_sharded(config, air, Untouchable(dev), None, [0, WIDTH])


# ---------------------------------------------------------------- proofs on the stand-in device
PROOF_CASES = [(c, rows) for c in ("poseidon2", "keccak") for rows in (1 << 3, 1 << 6)]
NUM_QUERIES, POW_BITS = 6, 3


def mock_prove(config_name, rows):
    """(proof, raw bytes, restated verifier config) of the BabyBear Poseidon2 AIR over `rows` rows on the stand-in device, under the
    Poseidon1 objective's configurations (tests/test_poseidon1_air_cpu.py)."""
    import keccak_transcript as K
    import stark_verify as V
    from test_poseidon1_air_cpu import p1_poseidon2_setup
    from plonky3_b200.uni_stark import prove
    mock = BabyBearP2MockGpu()
    if config_name == "keccak":
        config = K.keccak_mock_config(f, mock, NUM_QUERIES, POW_BITS)
        vcfg = K.verifier_config(f, NUM_QUERIES, POW_BITS)
    else:
        config, cfg = p1_poseidon2_setup(f, mock, NUM_QUERIES, POW_BITS)
        vcfg = V.product_config(f, cfg)
    air = PA.VectorizedPoseidon2Air(f, BO.example_constants(), mock)
    trace = air.generate_trace_rows(torch.from_numpy(_inputs(8 * rows, 7).view(np.int32)))
    proof = prove(config, air, trace)
    assert "p2air_quotient" in mock.calls
    return proof, proof.to_postcard(), vcfg


@pytest.mark.parametrize("config_name,rows", PROOF_CASES)
def test_proofs_on_the_stand_in_device(monkeypatch, config_name, rows):
    from test_keccak_air_cpu import corruption_sites
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import verify
    from plonky3_b200.verifier import VerificationError
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    proof, raw, vcfg = mock_prove(config_name, rows)
    assert proof.degree_bits == rows.bit_length() - 1 and len(proof.quotient_chunks) == 2
    assert proof.trace_next is None and len(proof.trace_local) == WIDTH
    verifier_air = PA.VectorizedPoseidon2Air(f, BO.example_constants(), None)
    verify(vcfg, verifier_air, raw)
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, verifier_air, bytes(bad))
    # an opened register that breaks its constraint is rejected at the out-of-domain check
    bad = proof.__class__.__new__(proof.__class__)
    bad.__dict__.update(proof.__dict__)
    bad.trace_local = np.array(proof.trace_local, dtype=np.uint32)
    col = 5 * COLS + 16 + 4 * 32 + 6                                    # permutation 5's fourth partial register
    bad.trace_local[col, 0] = (int(bad.trace_local[col, 0]) + 1) % f.P
    with pytest.raises(VerificationError):
        verify(vcfg, verifier_air, bad.to_postcard())
