"""The Blake3 AIR (plonky3_b200.blake3_air) without a GPU: its column layout, the restated compression (tests/blake3_air_oracle.py)
against the published BLAKE3 digests, the restated trace generation against that compression, the pinned random draw, the
constraint DAG (count, degree, vanishing on valid traces over both fields, corruptions in every part of the row), and proofs on
the oracle-backed stand-in device under both configurations, accepted by the product verifier and rejecting tampered bytes."""
import copy
import struct

import numpy as np
import pytest
import torch

import air_oracle as A
import blake3_air_oracle as BO
import mock_device as M
from plonky3_b200 import air as AIR
from plonky3_b200 import blake3_air as BA
from plonky3_b200.field import BabyBear, KoalaBear

FIELDS = [BabyBear, KoalaBear]
ALL_ONES = (1 << 32) - 1


def _inputs(n, seed):
    return np.random.default_rng(seed).integers(0, 1 << 32, (n, 24), dtype=np.uint32)


def _edge_inputs(n, seed):
    """Random inputs with row 0 all zeros and row 1 all ones (when there are such rows)."""
    x = _inputs(n, seed)
    x[0] = 0
    if n > 1:
        x[1] = ALL_ONES
    return x


class Blake3MockGpu(M.MockGpu):
    """The stand-in device with the Blake3 AIR's two calls: the trace from the restated generation, the quotient from the
    constraint-DAG oracle (tests/air_oracle.py) on the AIR's DAG."""

    def blake3_air_generate_trace(self, field, inputs):
        self._note("blake3_air_generate_trace")
        return M._t(BO.generate(field, inputs.contiguous().numpy().view(np.uint32)))

    def blake3_air_quotient(self, field, lde, log_trace_height, alpha):
        self._note("blake3_air_quotient")
        nodes, cons = BO.air_dag(BabyBear if field == BabyBear.id else KoalaBear)
        return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_trace_height + 1, log_trace_height, [], M._n(alpha)))


# ---------------------------------------------------------------- layout, compression, trace, constraints
def test_width_and_column_offsets():
    assert BA.WIDTH == 9168
    air = BA.Blake3Air(KoalaBear)
    assert air.width() == 9168 and air.num_public_values() == 0 and air.main_next_row_columns() == []
    assert (BA.INPUTS, BA.CHAINING_VALUES, BA.COUNTER_LOW, BA.COUNTER_HI, BA.BLOCK_LEN, BA.FLAGS) == (0, 512, 768, 800, 832, 864)
    assert (BA.INITIAL_ROW0, BA.INITIAL_ROW2, BA.FULL_ROUNDS, BA.FINAL_ROUND_HELPERS, BA.OUTPUTS) == (896, 904, 912, 8528, 8656)
    assert BA.state(6, BA.STATE_OUTPUT) + BA.STATE_WIDTH == BA.FINAL_ROUND_HELPERS == 912 + 7 * 4 * 272
    assert BA.outputs(3, 3, 31) == 9167 and BA.chaining_values(1, 3, 31) == 767 and BA.inputs(15, 31) == 511
    s = BA.state(0, BA.STATE_PRIME)
    assert (BA.row0(s, 3, 1), BA.row1(s, 3, 31), BA.row2(s, 3, 1), BA.row3(s, 3, 31)) == (919, 1047, 1055, 1183)
    # one row per hash: nothing reads the next row, and there are no selectors
    assert not any(n[0] in (AIR.MAIN_NEXT, AIR.IS_FIRST_ROW, AIR.IS_LAST_ROW, AIR.IS_TRANSITION) for n in air.nodes)


@pytest.mark.parametrize("field", FIELDS)
def test_constraint_count_and_degree(field):
    air = BA.Blake3Air(field)
    degs = air.constraint_degrees()
    assert len(degs) == 9632 and max(degs) == 3 and air.max_constraint_degree() == 3


def _digest(msg: bytes) -> str:
    """BLAKE3 of a message of at most one block: one compression with cv = IV, counter 0, CHUNK_START | CHUNK_END | ROOT."""
    block = np.array(struct.unpack("<16I", msg + bytes(64 - len(msg))), dtype=np.uint32)
    flags = BO.CHUNK_START | BO.CHUNK_END | BO.ROOT
    assert flags == 11
    out = BO.compress(np.array(BA.IV, dtype=np.uint32), block, 0, len(msg), flags)[0, :8]
    return struct.pack("<8I", *(int(w) for w in out)).hex()


def test_compression_reproduces_the_published_digests():
    assert _digest(b"") == "af1349b9f5f9a1a6a0404dea36dcc9499bcb25c9adc112b7cc9a93cae41f3262"
    assert _digest(b"abc") == "6437b3ac38465133ffb63b75273a8db548c558465d79db03fd359c6cd5bd9d85"


def test_message_schedule_is_the_permutation_iterated():
    assert BO.SCHEDULE[1] == BA.MSG_PERMUTATION
    assert BO.SCHEDULE[6] == [11, 15, 5, 0, 1, 9, 8, 6, 14, 10, 2, 12, 3, 4, 7, 13]


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 2, 8, 64])
def test_trace_outputs_are_the_compression_of_each_row(field, n):
    x = _edge_inputs(n, 30 + n)
    t = BO.generate(field.id, x)
    assert t.shape == (n, 9168) and np.all(t < field.P)
    exp = BO.compress(x[:, 16:], x[:, :16], np.arange(n, dtype=np.uint64), n, 0)
    assert np.array_equal(BO.output_words(field.id, t), exp)
    one = field.to_monty(1)
    bits = lambda w: [one if (int(w) >> i) & 1 else 0 for i in range(32)]
    r = n - 1
    assert list(t[r, BA.COUNTER_LOW:BA.COUNTER_LOW + 32]) == bits(r)
    assert list(t[r, BA.BLOCK_LEN:BA.BLOCK_LEN + 32]) == bits(n)
    assert not np.any(t[:, BA.COUNTER_HI:BA.COUNTER_HI + 32]) and not np.any(t[:, BA.FLAGS:BA.FLAGS + 32])


def test_generation_requires_a_power_of_two():
    with pytest.raises(AssertionError):
        BO.generate(KoalaBear.id, _inputs(3, 1))


def test_random_inputs_are_the_pinned_u32_draw():
    import fixture_replay as FR
    a = BA.random_inputs(5)
    assert a.shape == (5, 24) and a.dtype == np.uint32 and np.array_equal(a, BA.random_inputs(5))
    assert np.array_equal(BA.random_inputs(2), a[:2])
    rng = FR.SmallRng(1)
    assert [int(v) for v in a.ravel()] == [rng.u32() for _ in range(5 * 24)]


def _violated(field, tr):
    nodes, cons = BO.air_dag(field)
    return bool(np.any(BO.constraint_values(field.id, nodes, cons, tr)))


@pytest.mark.parametrize("field", FIELDS)
def test_constraints_vanish_on_valid_traces(field):
    for n, seed in ((1, 10), (8, 11)):
        assert not _violated(field, BO.generate(field.id, _edge_inputs(n, seed)))
    assert not _violated(field, BO.generate(field.id, np.full((2, 24), ALL_ONES, dtype=np.uint32)))


@pytest.mark.parametrize("field", FIELDS)
def test_corruptions_are_detected(field):
    one = field.to_monty(1)
    base = BO.generate(field.id, _edge_inputs(4, 5))

    def flip(v): return 0 if int(v) else one

    def add1(v): return field.to_monty((field.from_monty(int(v)) + 1) % field.P)
    sp, smp = BA.state(2, BA.STATE_PRIME), BA.state(4, BA.STATE_MIDDLE_PRIME)
    cases = [
        (BA.inputs(5, 7), flip), (BA.chaining_values(0, 2, 9), flip), (BA.chaining_values(1, 3, 30), flip),
        (BA.COUNTER_LOW + 1, flip), (BA.initial_row2(1, 0), add1), (BA.initial_row0(2, 1), add1),
        (BA.row0(sp, 1, 0), add1), (BA.row2(sp, 3, 1), add1), (BA.row3(smp, 2, 17), flip), (BA.row1(smp, 0, 3), flip),
        (BA.final_round_helpers(1, 4), flip),
    ] + [(BA.outputs(k, k, 3 + k), flip) for k in range(4)] + [
        (BA.inputs(0, 0), lambda v: field.to_monty(2)), (BA.row1(BA.state(3, BA.STATE_OUTPUT), 1, 1), lambda v: field.to_monty(2)),
    ]
    for col, fn in cases:
        for row in (0, 3):
            tr = base.copy()
            tr[row, col] = fn(tr[row, col])
            assert _violated(field, tr), (col, row)


# ---------------------------------------------------------------- proofs on the stand-in device
PROOF_CASES = [(f, c, n) for f in FIELDS for c in ("poseidon2", "keccak") for n in (1 << 5, 1 << 7)]
NUM_QUERIES, POW_BITS = 6, 3


def mock_prove(field, config_name, n_hashes):
    """(proof, raw bytes, product verifier config) of the Blake3 AIR on the stand-in device."""
    import keccak_transcript as K
    import stark_verify as V
    from test_keccak_air_cpu import poseidon2_setup
    from plonky3_b200.uni_stark import prove
    mock = Blake3MockGpu()
    if config_name == "keccak":
        config = K.keccak_mock_config(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = K.verifier_config(field, NUM_QUERIES, POW_BITS)
    else:
        config, cfg = poseidon2_setup(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = V.product_config(field, cfg)
    air = BA.Blake3Air(field, mock)
    trace = air.generate_trace_rows(torch.from_numpy(_edge_inputs(n_hashes, 7).view(np.int32)))
    proof = prove(config, air, trace)
    assert "blake3_air_quotient" in mock.calls
    return proof, proof.to_postcard(), vcfg


@pytest.mark.parametrize("field,config_name,n_hashes", PROOF_CASES)
def test_proofs_on_the_stand_in_device(monkeypatch, field, config_name, n_hashes):
    from test_keccak_air_cpu import corruption_sites
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import verify
    from plonky3_b200.verifier import VerificationError
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    proof, raw, vcfg = mock_prove(field, config_name, n_hashes)
    assert proof.degree_bits == n_hashes.bit_length() - 1 and len(proof.quotient_chunks) == 2
    assert proof.trace_next is None and len(proof.trace_local) == 9168
    verifier_air = BA.Blake3Air(field)                                # verifier-only: no device
    verify(vcfg, verifier_air, raw)
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, verifier_air, bytes(bad))
    # a proof whose opened row breaks a constraint is rejected at the out-of-domain check
    bad = copy.deepcopy(proof)
    bad.trace_local = np.array(bad.trace_local, dtype=np.uint32)
    col = BA.row1(BA.state(3, BA.STATE_MIDDLE), 2, 5)
    bad.trace_local[col, 0] = (int(bad.trace_local[col, 0]) + 1) % field.P
    with pytest.raises(VerificationError):
        verify(vcfg, verifier_air, bad.to_postcard())
