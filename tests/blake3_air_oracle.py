"""Oracle of the Blake3 AIR (plonky3_b200.blake3_air) — test infrastructure.

    compress(cv, block, counter, block_len, flags)   the BLAKE3 compression function (16 output words) restated in numpy,
                                 vectorised over rows: the known-answer tests pin it to the published BLAKE3 digests.
    generate(fid, inputs)        generate_trace_rows (blake3-air/src/generation.rs:16-118) restated in numpy: (n, 9168) Montgomery
                                 words, row i hashed with counter i, block_len n, flags 0.
    output_words(fid, trace)     the 16 output words of every row, decoded from the `outputs` bits.
    constraint_values(...)       the AIR's DAG on every row (keccak_air_oracle.constraint_values: check_constraints' semantics).
    air_dag(field)               the AIR's (nodes, constraints), built once per field.
"""
import numpy as np

from keccak_air_oracle import constraint_values  # noqa: F401  (the same DAG evaluator)
from plonky3_b200 import blake3_air as BA

_P = {0: 0x78000001, 1: 0x7F000001}
_U32 = np.uint32
CHUNK_START, CHUNK_END, ROOT = 1, 2, 8
SCHEDULE = [list(range(16))]
for _ in range(BA.NUM_ROUNDS - 1):
    SCHEDULE.append([SCHEDULE[-1][BA.MSG_PERMUTATION[i]] for i in range(16)])


def _rotr(v, r):
    return (v >> _U32(r)) | (v << _U32(32 - r))


def _half(v, a, b, c, d, m, second):
    r1, r2 = (8, 7) if second else (16, 12)
    v[a] = v[a] + v[b] + m
    v[d] = _rotr(v[d] ^ v[a], r1)
    v[c] = v[c] + v[d]
    v[b] = _rotr(v[b] ^ v[c], r2)


def _rounds(v, block, on_state=None):
    """The seven rounds on v (16 arrays of u32), in generation.rs's half-round order; on_state(r, s, v) after each of the four
    saved states of round r."""
    for r in range(BA.NUM_ROUNDS):
        m = [block[:, SCHEDULE[r][i]] for i in range(16)]
        for s, (diag, second) in enumerate(((False, False), (False, True), (True, False), (True, True))):
            for i in range(4):
                idx = (i, 4 + (i + diag) % 4, 8 + (i + 2 * diag) % 4, 12 + (i + 3 * diag) % 4)
                _half(v, *idx, m[8 * diag + 2 * i + second], second)
            if on_state:
                on_state(r, s, v)
    return v


def _initial(cv, counter, block_len, flags):
    n = cv.shape[0]
    full = lambda x: np.broadcast_to(np.asarray(x, dtype=np.uint64), (n,))
    ctr = full(counter)
    return ([cv[:, j].copy() for j in range(8)] + [np.full(n, BA.IV[j], _U32) for j in range(4)]
            + [(ctr & 0xFFFFFFFF).astype(_U32), (ctr >> np.uint64(32)).astype(_U32), full(block_len).astype(_U32), full(flags).astype(_U32)])


def compress(cv, block, counter, block_len, flags):
    """BLAKE3 compress: cv (n, 8), block (n, 16) u32, counter / block_len / flags scalars or (n,) -> (n, 16) u32 (the first 8
    words are the chaining value / digest words)."""
    cv = np.asarray(cv, dtype=_U32).reshape(-1, 8)
    block = np.asarray(block, dtype=_U32).reshape(-1, 16)
    with np.errstate(over="ignore"):
        v = _rounds(_initial(cv, counter, block_len, flags), block)
    return np.stack([v[j] ^ v[j + 8] for j in range(8)] + [v[j + 8] ^ cv[:, j] for j in range(8)], axis=1)


def _bits(fid, w):
    """(n, 32) Montgomery 0 / 1 of u32 words, least significant first."""
    one = (1 << 32) % _P[fid]
    bits = ((w[:, None] >> np.arange(32, dtype=_U32)) & _U32(1)).astype(np.uint64)
    return (bits * np.uint64(one)).astype(np.uint32)


def _limbs(fid, w):
    """(n, 2) Montgomery [lo, hi] 16-bit limbs of u32 words."""
    one = (1 << 32) % _P[fid]
    v = np.stack([w & _U32(0xFFFF), w >> _U32(16)], axis=1).astype(np.uint64)
    return (v * np.uint64(one) % np.uint64(_P[fid])).astype(np.uint32)


def generate(fid, inputs):
    """(n, 24) u32 inputs (16 message words, 8 chaining-value words), n a power of two -> (n, 9168) Montgomery trace."""
    n = np.asarray(inputs).reshape(-1, 24).shape[0]
    assert n > 0 and n & (n - 1) == 0, "the number of inputs must be a power of two"
    return generate_rows(fid, inputs, 0, n)


def generate_rows(fid, inputs, first_row, n_rows):
    """Rows [first_row, first_row + len(inputs)) of the trace of an n_rows-row trace: a row depends on its input, its index (the
    counter) and the row count (block_len) only."""
    inputs = np.ascontiguousarray(inputs, dtype=_U32).reshape(-1, 24)
    n = inputs.shape[0]
    t = np.zeros((n, BA.WIDTH), dtype=np.uint32)

    def put_bits(col, w): t[:, col:col + 32] = _bits(fid, w)

    def put_state(base, v):
        for j in range(4):
            t[:, BA.row0(base, j, 0):BA.row0(base, j, 0) + 2] = _limbs(fid, v[j])
            put_bits(BA.row1(base, j, 0), v[4 + j])
            t[:, BA.row2(base, j, 0):BA.row2(base, j, 0) + 2] = _limbs(fid, v[8 + j])
            put_bits(BA.row3(base, j, 0), v[12 + j])

    block, cv = inputs[:, :16], inputs[:, 16:]
    counter = np.arange(first_row, first_row + n, dtype=np.uint64)
    for w in range(16):
        put_bits(BA.inputs(w, 0), block[:, w])
    for j in range(8):
        put_bits(BA.CHAINING_VALUES + 32 * j, cv[:, j])
    v = _initial(cv, counter, n_rows, 0)
    for base, w in zip((BA.COUNTER_LOW, BA.COUNTER_HI, BA.BLOCK_LEN, BA.FLAGS), v[12:]):
        put_bits(base, w)
    for j in range(4):
        t[:, BA.initial_row0(j, 0):BA.initial_row0(j, 0) + 2] = _limbs(fid, cv[:, j])
        t[:, BA.initial_row2(j, 0):BA.initial_row2(j, 0) + 2] = _limbs(fid, np.full(n, BA.IV[j], _U32))
    with np.errstate(over="ignore"):
        v = _rounds(v, block, lambda r, s, v: put_state(BA.state(r, s), v))
    for j in range(4):
        put_bits(BA.final_round_helpers(j, 0), v[8 + j])
        put_bits(BA.outputs(0, j, 0), v[j] ^ v[8 + j])
        put_bits(BA.outputs(1, j, 0), v[4 + j] ^ v[12 + j])
        put_bits(BA.outputs(2, j, 0), v[8 + j] ^ cv[:, j])
        put_bits(BA.outputs(3, j, 0), v[12 + j] ^ cv[:, 4 + j])
    return t


def output_words(fid, trace):
    """(n, 16) u32: the `outputs` bits of every row, packed (outputs[k][j] is output word 4 k + j)."""
    p = _P[fid]
    bits = np.asarray(trace[:, BA.OUTPUTS:BA.OUTPUTS + 512], dtype=np.uint32).reshape(-1, 16, 32)
    one = (1 << 32) % p
    assert np.all((bits == 0) | (bits == one))
    return ((bits == one).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


_DAGS = {}


def air_dag(field):
    """(nodes (n, 4) uint32, constraints) of Blake3Air over `field`."""
    if field.id not in _DAGS:
        air = BA.Blake3Air(field)
        _DAGS[field.id] = (air.nodes, air.constraints)
    return _DAGS[field.id]
