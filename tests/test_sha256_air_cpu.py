"""The SHA-256 AIR (plonky3_b200.sha256_air) without a GPU: its column layout and constraint order, the restated compression
(tests/sha256_air_oracle.py) against hashlib.sha256 and a plain Python compression, the restated trace generation against that
compression, the pinned random draw, the constraint DAG (count, degree, vanishing on valid traces over both fields, corruptions in
every column class), the KernelAir guards, and proofs on the oracle-backed stand-in device under both configurations, accepted by
the product verifier and rejecting tampered bytes."""
import copy
import hashlib
import struct

import numpy as np
import pytest
import torch

import air_oracle as A
import mock_device as M
import sha256_air_oracle as SO
from plonky3_b200 import _lib
from plonky3_b200 import air as AIR
from plonky3_b200 import sha256_air as SA
from plonky3_b200.field import BabyBear, KoalaBear

FIELDS = [BabyBear, KoalaBear]
ALL_ONES = (1 << 32) - 1


def _inputs(n, seed):
    return np.random.default_rng(seed).integers(0, 1 << 32, (n, 24), dtype=np.uint32)


def boundary_inputs():
    """The reference's boundary rows (check_constraints_pass_at_boundary_values): block and state 0; block and state 2^32 - 1; a
    walking 1-bit block on the IV; the IV padded to 16 words as the block, on the IV."""
    iv = list(SO.IV)
    return np.array([[0] * 24, [ALL_ONES] * 24, [1 << (i % 32) for i in range(16)] + iv, iv + [0] * 8 + iv], dtype=np.uint32)


def _edge_inputs(n, seed):
    """Random inputs whose first rows (as many as fit) are the reference's boundary rows."""
    x = _inputs(n, seed)
    b = boundary_inputs()
    x[:min(n, 4)] = b[:min(n, 4)]
    return x


class Sha256MockGpu(M.MockGpu):
    """The stand-in device with the SHA-256 AIR's two calls: the trace from the restated generation, the quotient from the
    constraint-DAG oracle (tests/air_oracle.py) on the AIR's DAG."""

    def sha256_air_generate_trace(self, field, inputs):
        self._note("sha256_air_generate_trace")
        return M._t(SO.generate(field, inputs.contiguous().numpy().view(np.uint32)))

    def sha256_air_quotient(self, field, lde, log_trace_height, alpha):
        self._note("sha256_air_quotient")
        nodes, cons = SO.air_dag(BabyBear if field == BabyBear.id else KoalaBear)
        return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_trace_height + 1, log_trace_height, [], M._n(alpha)))


# ---------------------------------------------------------------- layout and constraint order
def test_width_and_column_offsets():
    # Sha256Cols' fields in declaration order, sized from columns.rs / constants.rs
    sizes = [("h_in", 8 * 2), ("a_chain", 68 * 32), ("e_chain", 68 * 32), ("w", 64 * 32), ("sched_sigma0", 48 * 2),
             ("sched_sigma1", 48 * 2), ("sched_tmp", 48 * 2), ("rounds", 64 * 6 * 2), ("h_out", 8 * 32)]
    offsets = dict(zip([s[0] for s in sizes], np.cumsum([0] + [s[1] for s in sizes])[:-1].tolist()))
    assert offsets == {"h_in": SA.H_IN, "a_chain": SA.A_CHAIN, "e_chain": SA.E_CHAIN, "w": SA.W, "sched_sigma0": SA.SCHED_SIGMA0,
                       "sched_sigma1": SA.SCHED_SIGMA1, "sched_tmp": SA.SCHED_TMP, "rounds": SA.ROUNDS, "h_out": SA.H_OUT}
    assert (SA.A_CHAIN, SA.E_CHAIN, SA.W, SA.SCHED_SIGMA0, SA.ROUNDS, SA.H_OUT) == (16, 2192, 4368, 6416, 6704, 7472)
    assert SA.WIDTH == sum(s[1] for s in sizes) == 7728 and SA.WIDTH % 16 == 0 and SA.WIDTH < 8192
    air = SA.Sha256Air(KoalaBear)
    assert air.width() == 7728 and air.num_public_values() == 0 and air.main_next_row_columns() == []
    assert SA.rounds(63, SA.MAJ, 1) == SA.H_OUT - 1 and SA.h_out(7, 31) == 7727 and SA.e_chain(67, 31) == SA.W - 1
    # one row per hash: nothing reads the next row, and there are no selectors or public values
    assert not any(n[0] in (AIR.MAIN_NEXT, AIR.IS_FIRST_ROW, AIR.IS_LAST_ROW, AIR.IS_TRANSITION, AIR.PUBLIC) for n in air.nodes)


def test_round_constants_and_iv_are_the_standard_ones():
    assert SA.K == SO.K and SA.IV == SO.IV


@pytest.mark.parametrize("field", FIELDS)
def test_constraint_count_and_degree(field):
    air = SA.Sha256Air(field)
    degs = air.constraint_degrees()
    assert len(degs) == 8096 and max(degs) == 3 and air.max_constraint_degree() == 3


def _cone_columns(nodes, root):
    """The trace columns constraint node `root` reads."""
    cols, stack, seen = set(), [int(root)], set()
    while stack:
        i = stack.pop()
        if i in seen:
            continue
        seen.add(i)
        op, a, b, _ = (int(v) for v in nodes[i])
        if op == AIR.MAIN_LOCAL:
            cols.add(a)
        elif op in (AIR.ADD, AIR.SUB, AIR.MUL):
            stack += [a, b]
        elif op == AIR.NEG:
            stack.append(a)
    return cols


def test_constraint_order_is_the_reference_s_emission_order():
    nodes, cons = SO.air_dag(KoalaBear)
    word = lambda col: set(range(col, col + 32))
    lo16 = lambda col: set(range(col, col + 16))
    cone = lambda k: _cone_columns(nodes, cons[k])
    # booleans of w, a_chain, e_chain, h_out (not column order)
    for k, col in ((0, SA.w(0, 0)), (2047, SA.w(63, 31)), (2048, SA.a_chain(0, 0)), (4223, SA.a_chain(67, 31)),
                   (4224, SA.e_chain(0, 0)), (6399, SA.e_chain(67, 31)), (6400, SA.h_out(0, 0)), (6655, SA.h_out(7, 31))):
        assert cone(k) == {col}, k
    # h_in against chain slots 3..0, a then e
    assert cone(6656) == {SA.h_in(0, 0)} | lo16(SA.a_chain(3, 0))
    assert cone(6671) == {SA.h_in(7, 1)} | lo16(SA.e_chain(0, 16))
    # schedule step 0 opens with small sigma0's low limb: bits i + 7, i + 18 (mod 32) and i + 3 (a shift) of w[1], i < 16
    assert cone(6672) == {SA.sched_sigma0(0, 0)} | {SA.w(1, (i + r) % 32) for i in range(16) for r in (7, 18)} | {
        SA.w(1, i + 3) for i in range(16)}
    # small sigma1's high limb: bit i + 10 of a shift reads zero past bit 31
    assert cone(6675) == {SA.sched_sigma1(0, 1)} | {SA.w(14, (i + r) % 32) for i in range(16, 32) for r in (17, 19)} | {
        SA.w(14, i + 10) for i in range(16, 22)}
    # step 47 closes with add3_expr_out(pack(w[63]), sched_tmp, sched_sigma0, pack(w[47])): the 2^32 check, then the 2^16 check
    assert cone(7054) == word(SA.w(63, 0)) | word(SA.w(47, 0)) | {SA.sched_tmp(47, 0), SA.sched_tmp(47, 1), SA.sched_sigma0(47, 0),
                                                                   SA.sched_sigma0(47, 1)}
    assert cone(7055) == lo16(SA.w(63, 0)) | lo16(SA.w(47, 0)) | {SA.sched_tmp(47, 0), SA.sched_sigma0(47, 0)}
    # round 0 starts with sigma1 of e = e_chain[3]; round 63 ends with new_e = d + t1 (d = a_chain[63])
    assert cone(7056) == {SA.rounds(0, SA.SIGMA1_E, 0)} | {SA.e_chain(3, (i + r) % 32) for i in range(16) for r in (6, 11, 25)}
    assert cone(8078) == word(SA.e_chain(67, 0)) | word(SA.a_chain(63, 0)) | {SA.rounds(63, SA.T1, 0), SA.rounds(63, SA.T1, 1)}
    assert cone(8079) == lo16(SA.e_chain(67, 0)) | lo16(SA.a_chain(63, 0)) | {SA.rounds(63, SA.T1, 0)}
    # finalization: h_out[0] = h_in[0] + a_chain[67], ..., h_out[7] = h_in[7] + e_chain[64]
    assert cone(8080) == word(SA.h_out(0, 0)) | word(SA.a_chain(67, 0)) | {SA.h_in(0, 0), SA.h_in(0, 1)}
    assert cone(8095) == lo16(SA.h_out(7, 0)) | lo16(SA.e_chain(64, 0)) | {SA.h_in(7, 0)}


# ---------------------------------------------------------------- the compression and the trace
def _py_compress(h, block):
    """A plain Python SHA-256 compression (FIPS 180-4 section 6.2.2), independent of the numpy restatement."""
    rotr = lambda x, r: ((x >> r) | (x << (32 - r))) & ALL_ONES
    wv = list(block)
    for t in range(16, 64):
        s0 = rotr(wv[t - 15], 7) ^ rotr(wv[t - 15], 18) ^ (wv[t - 15] >> 3)
        s1 = rotr(wv[t - 2], 17) ^ rotr(wv[t - 2], 19) ^ (wv[t - 2] >> 10)
        wv.append((wv[t - 16] + s0 + wv[t - 7] + s1) & ALL_ONES)
    a, b, c, d, e, f, g, hh = h
    for t in range(64):
        t1 = (hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + SO.K[t] + wv[t]) & ALL_ONES
        t2 = ((rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c))) & ALL_ONES
        a, b, c, d, e, f, g, hh = (t1 + t2) & ALL_ONES, a, b, c, (d + t1) & ALL_ONES, e, f, g
    return [(x + y) & ALL_ONES for x, y in zip(h, (a, b, c, d, e, f, g, hh))]


def _sha256(msg: bytes) -> str:
    """SHA-256 of msg through the restated compression: pad, then chain the blocks from the IV."""
    padded = msg + b"\x80" + bytes((55 - len(msg)) % 64) + struct.pack(">Q", 8 * len(msg))
    h = np.array(SO.IV, dtype=np.uint32)
    for off in range(0, len(padded), 64):
        h = SO.compress(h, np.array(struct.unpack(">16I", padded[off:off + 64]), dtype=np.uint32))[0]
    return struct.pack(">8I", *(int(x) for x in h)).hex()


@pytest.mark.parametrize("msg", [b"", b"abc", b"x" * 55])
def test_compression_reproduces_hashlib_for_one_block(msg):
    assert _sha256(msg) == hashlib.sha256(msg).hexdigest()


@pytest.mark.parametrize("msg", [b"x" * 56, b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq", bytes(range(119))])
def test_compression_reproduces_hashlib_for_two_blocks(msg):
    assert (len(msg) + 9 + 63) // 64 == 2
    assert _sha256(msg) == hashlib.sha256(msg).hexdigest()


@pytest.mark.parametrize("block,state", [([0] * 16, SO.IV), ([ALL_ONES] * 16, [ALL_ONES] * 8)])
def test_compression_matches_the_reference_test_cases(block, state):
    got = SO.compress(np.array(state, dtype=np.uint32), np.array(block, dtype=np.uint32))[0]
    assert [int(x) for x in got] == _py_compress(list(state), block)


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 4, 16])
def test_trace_outputs_are_the_compression_of_each_row(field, n):
    x = _edge_inputs(n, 30 + n)
    t = SO.generate(field.id, x)
    assert t.shape == (n, 7728) and np.all(t < field.P)
    assert np.array_equal(SO.output_words(field.id, t), SO.compress(x[:, 16:], x[:, :16]))
    for r in range(n):
        assert [int(v) for v in SO.output_words(field.id, t[r:r + 1])[0]] == _py_compress([int(v) for v in x[r, 16:]],
                                                                                         [int(v) for v in x[r, :16]])
    one = field.to_monty(1)
    bits = lambda v: [one if (int(v) >> i) & 1 else 0 for i in range(32)]
    r = n - 1
    assert [field.from_monty(int(v)) for v in t[r, :16]] == [int(x[r, 16 + i // 2]) >> (16 * (i & 1)) & 0xFFFF for i in range(16)]
    assert list(t[r, SA.a_chain(0, 0):SA.a_chain(1, 0)]) == bits(x[r, 16 + 3])          # a_chain[0] = H3
    assert list(t[r, SA.e_chain(3, 0):SA.e_chain(4, 0)]) == bits(x[r, 16 + 4])          # e_chain[3] = H4
    assert list(t[r, SA.w(15, 0):SA.w(16, 0)]) == bits(x[r, 15])


def test_generation_requires_a_power_of_two():
    with pytest.raises(AssertionError):
        SO.generate(KoalaBear.id, _inputs(3, 1))


def test_random_inputs_are_the_pinned_u32_draw():
    import fixture_replay as FR
    a = SA.random_inputs(5)
    assert a.shape == (5, 24) and a.dtype == np.uint32 and np.array_equal(a, SA.random_inputs(5))
    rng = FR.SmallRng(1)
    assert [int(v) for v in a.ravel()] == [rng.u32() for _ in range(5 * 24)]


def _violated_rows(field, tr):
    nodes, cons = SO.air_dag(field)
    return np.any(SO.constraint_values(field.id, nodes, cons, tr), axis=0)


@pytest.mark.parametrize("field", FIELDS)
def test_constraints_vanish_on_valid_traces(field):
    tr = np.concatenate([SO.generate(field.id, boundary_inputs()), SO.generate(field.id, _inputs(4, 11))])
    assert not np.any(_violated_rows(field, tr))


@pytest.mark.parametrize("field", FIELDS)
def test_corruptions_are_detected(field):
    one = field.to_monty(1)
    base = SO.generate(field.id, boundary_inputs())

    def flip(v): return 0 if int(v) else one

    def add1(v): return field.to_monty((field.from_monty(int(v)) + 1) % field.P)

    def two(v): return field.to_monty(2)
    cases = [
        (SA.h_out(7, 31), flip), (SA.h_out(2, 5), flip),                     # a flipped output bit
        (SA.w(16, 0), flip), (SA.w(40, 13), flip), (SA.w(3, 31), flip),     # a flipped schedule bit (expanded and block words)
        (SA.h_out(0, 0), two), (SA.w(20, 7), two),                          # non-boolean bits
        (SA.a_chain(2, 9), flip), (SA.a_chain(40, 30), flip), (SA.e_chain(0, 1), flip), (SA.e_chain(67, 4), flip),   # chain bits
        (SA.a_chain(10, 3), two), (SA.e_chain(66, 22), two),
        (SA.h_in(1, 0), add1), (SA.h_in(6, 1), add1),                       # every packed family
        (SA.sched_sigma0(5, 1), add1), (SA.sched_sigma1(30, 0), add1), (SA.sched_tmp(47, 1), add1),
    ] + [(SA.rounds(7 * j + 3, fld, j & 1), add1) for j, fld in enumerate((SA.SIGMA1_E, SA.CH, SA.TMP1, SA.T1, SA.SIGMA0_A, SA.MAJ))]
    rows = []
    for col, fn in cases:
        for r in range(4):
            row = base[r].copy()
            row[col] = fn(row[col])
            rows.append(row)
    bad = _violated_rows(field, np.stack(rows))
    assert bad.shape == (4 * len(cases),)
    missed = [cases[i // 4][0] for i in np.flatnonzero(~bad)]
    assert not missed, missed


# ---------------------------------------------------------------- KernelAir guards
class _RecordingGpu:
    device = None

    def __init__(self):
        self.calls = []

    def sha256_air_quotient(self, *args):
        self.calls.append(args)
        return "quotient"


ALPHA = np.array([3, 5, 7, 11], dtype=np.uint32)


def test_guards_refuse_before_any_device_call():
    gpu = _RecordingGpu()
    air = SA.Sha256Air(KoalaBear, gpu)
    with pytest.raises(ValueError, match="^1 public values given, the SHA-256 AIR has none$"):
        air.quotient_values(object(), 4, ALPHA, public_values=[1])
    with pytest.raises(ValueError, match="^the SHA-256 AIR has no preprocessed columns$"):
        air.quotient_values(object(), 4, ALPHA, preprocessed_on_quotient_domain=object())
    assert gpu.calls == []
    with pytest.raises(_lib.P3GpuError, match="quotient evaluation needs a GPU context"):
        SA.Sha256Air(KoalaBear).quotient_values(object(), 4, ALPHA)
    with pytest.raises(_lib.P3GpuError, match="trace generation needs a GPU context"):
        SA.Sha256Air(KoalaBear).generate_random_trace_rows(4)
    lde = object()
    assert air.quotient_values(lde, 4, ALPHA) == "quotient"
    assert gpu.calls == [(KoalaBear.id, lde, 4, ALPHA)]


# ---------------------------------------------------------------- proofs on the stand-in device
PROOF_CASES = [(f, c, n) for f in FIELDS for c in ("poseidon2", "keccak") for n in (1 << 2, 1 << 5)]
NUM_QUERIES, POW_BITS = 6, 3


def mock_prove(field, config_name, n_hashes):
    """(proof, raw bytes, product verifier config) of the SHA-256 AIR on the stand-in device."""
    import keccak_transcript as K
    import stark_verify as V
    from test_keccak_air_cpu import poseidon2_setup
    from plonky3_b200.uni_stark import prove
    mock = Sha256MockGpu()
    if config_name == "keccak":
        config = K.keccak_mock_config(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = K.verifier_config(field, NUM_QUERIES, POW_BITS)
    else:
        config, cfg = poseidon2_setup(field, mock, NUM_QUERIES, POW_BITS)
        vcfg = V.product_config(field, cfg)
    air = SA.Sha256Air(field, mock)
    trace = air.generate_trace_rows(torch.from_numpy(_edge_inputs(n_hashes, 7).view(np.int32)))
    proof = prove(config, air, trace)
    assert "sha256_air_quotient" in mock.calls
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
    assert proof.trace_next is None and len(proof.trace_local) == 7728
    verifier_air = SA.Sha256Air(field)                                  # verifier-only: no device
    verify(vcfg, verifier_air, raw)
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, verifier_air, bytes(bad))
    # a proof whose opened row breaks a constraint is rejected at the out-of-domain check
    bad = copy.deepcopy(proof)
    bad.trace_local = np.array(bad.trace_local, dtype=np.uint32)
    col = SA.rounds(20, SA.T1, 0)
    bad.trace_local[col, 0] = (int(bad.trace_local[col, 0]) + 1) % field.P
    with pytest.raises(VerificationError):
        verify(vcfg, verifier_air, bad.to_postcard())
