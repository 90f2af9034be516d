"""Oracle of the Poseidon1 AIR (plonky3_b200.poseidon1_air) — test infrastructure, vectorised numpy on canonical int64:

    textbook     poseidon1/src/lib.rs: RF / 2 full rounds (AddRoundConstants, S-box on every element, dense circulant MDS), RP
                 partial rounds (AddRoundConstants, S-box on state[0], dense MDS), RF / 2 full rounds
    generation   poseidon1-air/src/generation.rs generate_trace_rows_for_perm: the optimized (sparse) form, one permutation ->
                 its columns, a row of vector_len permutations side by side (Montgomery words)
    constraints  keccak_air_oracle.constraint_values on the AIR's DAG
"""
import json
import pathlib

import numpy as np

from plonky3_b200 import poseidon1_air as PA
from plonky3_b200.field import BabyBear, KoalaBear

FIXTURE = pathlib.Path(__file__).resolve().parent / "golden" / "poseidon1_constants.json"
_KEY = {BabyBear.id: "baby_bear", KoalaBear.id: "koala_bear"}


def fixture(field):
    return json.loads(FIXTURE.read_text())[_KEY[field.id]]


def raw_constants(field) -> PA.Poseidon1Constants:
    return PA.Poseidon1Constants.from_fixture(field, fixture(field))


_OPT = {}


def optimized(field):
    """(FullRoundConstants, PartialRoundConstants) of the fixture's instance, cached."""
    if field.id not in _OPT:
        _OPT[field.id] = raw_constants(field).to_optimized()
    return _OPT[field.id]


def _sbox(field, x):
    p = field.P
    x2 = x * x % p
    x3 = x2 * x % p
    return x3 if field.SBOX_D == 3 else x3 * x3 % p * x % p


def _matvec(m, s, p):
    """(n, 16) states times the 16 x 16 matrix m: out[:, i] = sum_j m[i][j] s[:, j]."""
    out = np.zeros_like(s)
    for i in range(16):
        acc = np.zeros(s.shape[0], dtype=np.int64)
        for j in range(16):
            acc = (acc + int(m[i][j]) * s[:, j]) % p
        out[:, i] = acc
    return out


def textbook(field, raw: PA.Poseidon1Constants, states):
    """(n, 16) canonical -> the permuted (n, 16) canonical states."""
    p, half = field.P, raw.rounds_f // 2
    s = np.asarray(states, dtype=np.int64) % p
    mds = raw.dense_mds()
    rc = [np.array(r, dtype=np.int64) % p for r in raw.round_constants]
    for r in range(raw.rounds_f + raw.rounds_p):
        s = (s + rc[r]) % p
        if half <= r < half + raw.rounds_p:
            s[:, 0] = _sbox(field, s[:, 0])
        else:
            s = _sbox(field, s)
        s = _matvec(mds, s, p)
    return s


def optimized_permutation(field, full, partial, states):
    """The optimized form (poseidon1/src/lib.rs Poseidon1::permute_mut with the sparse partial rounds), canonical."""
    return _run(field, full, partial, np.asarray(states, dtype=np.int64) % field.P, None)


def _run(field, full, partial, s, put):
    """The optimized permutation of (n, 16) canonical states; put(values (n, k)) receives the committed columns in order."""
    p, reg = field.P, PA.sbox_registers(field)
    emit = put if put is not None else (lambda v: None)
    mds = PA.circulant([int(v) for v in full.mds_circ_col], p)

    def sbox(x):
        x3 = x * x % p * x % p
        if reg == 0:
            return x3, []
        return x3 * x3 % p * x % p, [x3]

    def full_round(s, rc):
        s = (s + np.asarray(rc, dtype=np.int64)) % p
        outs, regs = [], []
        for i in range(16):
            o, r = sbox(s[:, i])
            outs.append(o); regs += r
        if regs:
            emit(np.stack(regs, axis=1))
        s = _matvec(mds, np.stack(outs, axis=1), p)
        emit(s)
        return s
    emit(s)
    for rc in full.initial:
        s = full_round(s, rc)
    s = (s + np.asarray(partial.first_round_constants, dtype=np.int64)) % p
    s = _matvec(partial.m_i, s, p)
    rp = partial.rounds_p
    for r in range(rp):
        o, regs = sbox(s[:, 0])
        emit(np.stack(regs + [o], axis=1))
        s0 = o if r == rp - 1 else (o + int(partial.round_constants[r])) % p
        new0 = s0 * int(partial.sparse_first_row[r][0]) % p
        for j in range(1, 16):
            new0 = (new0 + s[:, j] * int(partial.sparse_first_row[r][j])) % p
        s = s.copy()
        for i in range(1, 16):
            s[:, i] = (s[:, i] + s0 * int(partial.v[r][i - 1])) % p
        s[:, 0] = new0
    for rc in full.terminal:
        s = full_round(s, rc)
    return s


def generate(field, full, partial, inputs, vector_len=PA.VECTOR_LEN):
    """generate_vectorized_trace_rows: (n, 16) Montgomery inputs, n = vector_len * 2^k -> (n / vector_len, vector_len * columns)
    Montgomery trace."""
    x = np.ascontiguousarray(inputs, dtype=np.uint32).reshape(-1, 16)
    n = x.shape[0]
    assert n % vector_len == 0 and (n // vector_len) & (n // vector_len - 1) == 0 and n > 0, \
        "the number of inputs must be vector_len times a power of two"
    return generate_perms(field, full, partial, x).reshape(n // vector_len, -1)


def generate_perms(field, full, partial, inputs):
    """(n, 16) Montgomery inputs -> (n, columns) Montgomery: every permutation's columns (no shape condition)."""
    parts = []
    _run(field, full, partial, field.from_monty_array(inputs).astype(np.int64), parts.append)
    t = np.concatenate(parts, axis=1)
    assert t.shape[1] == PA.columns(field, partial.rounds_p)
    return field.to_monty_array(t)


def last_post(field, partial, trace_perms):
    """(n, 16) canonical: every permutation's last `post` (the permutation's output), from (n, columns) Montgomery rows."""
    return field.from_monty_array(np.asarray(trace_perms)[:, -16:]).astype(np.int64)


_DAGS = {}


def air_dag(field, vector_len=PA.VECTOR_LEN):
    """(nodes (n, 4) uint32, constraints) of the fixture's VectorizedPoseidon1Air over `field`."""
    key = (field.id, vector_len)
    if key not in _DAGS:
        air = PA.VectorizedPoseidon1Air(field, optimized(field), vector_len=vector_len)
        _DAGS[key] = (air.nodes, air.constraints)
    return _DAGS[key]
