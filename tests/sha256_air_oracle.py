"""Oracle of the SHA-256 AIR (plonky3_b200.sha256_air) — test infrastructure.

    compress(h, block)           the SHA-256 compression function (FIPS 180-4 section 6.2.2) restated in numpy, vectorised over
                                 rows: the tests pin it to hashlib.sha256 and to a plain Python compression.
    generate(fid, inputs)        generate_trace_rows (sha256-air/src/generation.rs) restated in numpy, column by column: (n, 7728)
                                 Montgomery words.
    generate_rows(fid, inputs)   the same rows without the power-of-two check (a row depends on its own input only).
    output_words(fid, trace)     the 8 output words of every row, decoded from the `h_out` bits.
    constraint_values(...)       the AIR's DAG on every row (keccak_air_oracle.constraint_values: check_constraints' semantics).
    air_dag(field)               the AIR's (nodes, constraints), built once per field.

Only the column offsets are taken from plonky3_b200.sha256_air (the CPU test checks them against the struct's field sizes); the
round constants are restated here.
"""
import numpy as np

from keccak_air_oracle import constraint_values  # noqa: F401  (the same DAG evaluator)
from plonky3_b200 import sha256_air as SA

_P = {0: 0x78000001, 1: 0x7F000001}
_U32 = np.uint32
# FIPS 180-4 section 4.2.2: the first 32 bits of the fractional parts of the cube roots of the first 64 primes
_PRIMES = [p for p in range(2, 312) if all(p % d for d in range(2, int(p ** 0.5) + 1))][:64]


def _frac_root_bits(p, k):
    """floor(2^32 * frac(p^(1/k))), exactly: the largest x with x^k <= p * 2^(32 k), minus the integer part."""
    target = p << (32 * k)
    lo, hi = 0, 1 << 40
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if mid ** k <= target else (lo, mid - 1)
    return lo & 0xFFFFFFFF


K = [_frac_root_bits(p, 3) for p in _PRIMES]
IV = [_frac_root_bits(p, 2) for p in _PRIMES[:8]]        # section 5.3.3: square roots of the first 8 primes


def _rotr(v, r):
    return (v >> _U32(r)) | (v << _U32(32 - r))


def _schedule(block):
    """The 64 schedule words and the per-step small sigma0, small sigma1 and sigma1 + w[t - 7] (lists of (n,) arrays)."""
    wv = [block[:, t].copy() for t in range(16)]
    s0s, s1s, tmps = [], [], []
    for t in range(16, 64):
        x15, x2 = wv[t - 15], wv[t - 2]
        s0 = _rotr(x15, 7) ^ _rotr(x15, 18) ^ (x15 >> _U32(3))
        s1 = _rotr(x2, 17) ^ _rotr(x2, 19) ^ (x2 >> _U32(10))
        tmp = s1 + wv[t - 7]
        wv.append(tmp + s0 + wv[t - 16])
        s0s.append(s0); s1s.append(s1); tmps.append(tmp)
    return wv, s0s, s1s, tmps


def _rounds(h, wv, on_round=None):
    """The 64 rounds from the state h (8 arrays); on_round(t, sigma1_e, ch, tmp1, t1, sigma0_a, maj, new_a, new_e) after each."""
    a, b, c, d, e, f, g, hh = h
    for t in range(64):
        s1e = _rotr(e, 6) ^ _rotr(e, 11) ^ _rotr(e, 25)
        ch = (e & f) ^ (~e & g)
        tmp1 = hh + s1e + ch
        t1 = tmp1 + _U32(K[t]) + wv[t]
        s0a = _rotr(a, 2) ^ _rotr(a, 13) ^ _rotr(a, 22)
        maj = (a & b) ^ (a & c) ^ (b & c)
        na, ne = t1 + s0a + maj, d + t1
        if on_round:
            on_round(t, s1e, ch, tmp1, t1, s0a, maj, na, ne)
        a, b, c, d, e, f, g, hh = na, a, b, c, ne, e, f, g
    return [a, b, c, d, e, f, g, hh]


def compress(h, block):
    """SHA-256 compress: h (n, 8), block (n, 16) u32 -> (n, 8) u32, the next chaining state."""
    h = np.asarray(h, dtype=_U32).reshape(-1, 8)
    block = np.asarray(block, dtype=_U32).reshape(-1, 16)
    with np.errstate(over="ignore"):
        fin = _rounds([h[:, j].copy() for j in range(8)], _schedule(block)[0])
        return np.stack([h[:, j] + fin[j] for j in range(8)], axis=1)


def _bits(fid, v):
    """(n, 32) Montgomery 0 / 1 of u32 words, least significant first."""
    one = (1 << 32) % _P[fid]
    bits = ((v[:, None] >> np.arange(32, dtype=_U32)) & _U32(1)).astype(np.uint64)
    return (bits * np.uint64(one)).astype(np.uint32)


def _limbs(fid, v):
    """(n, 2) Montgomery [lo, hi] 16-bit limbs of u32 words."""
    one = (1 << 32) % _P[fid]
    x = np.stack([v & _U32(0xFFFF), v >> _U32(16)], axis=1).astype(np.uint64)
    return (x * np.uint64(one) % np.uint64(_P[fid])).astype(np.uint32)


def generate(fid, inputs):
    """(n, 24) u32 inputs (the 16-word block, then the 8-word chaining state), n a power of two -> (n, 7728) Montgomery trace."""
    n = np.asarray(inputs).reshape(-1, 24).shape[0]
    assert n > 0 and n & (n - 1) == 0, "the number of inputs must be a power of two"
    return generate_rows(fid, inputs)


def generate_rows(fid, inputs):
    """The trace rows of `inputs`, one per input."""
    inputs = np.ascontiguousarray(inputs, dtype=_U32).reshape(-1, 24)
    n = inputs.shape[0]
    t = np.zeros((n, SA.WIDTH), dtype=np.uint32)
    block, h = inputs[:, :16], inputs[:, 16:]

    def put_bits(col, v): t[:, col:col + 32] = _bits(fid, v)

    def put_limbs(col, v): t[:, col:col + 2] = _limbs(fid, v)

    for i in range(8):
        put_limbs(SA.h_in(i, 0), h[:, i])
    with np.errstate(over="ignore"):
        wv, s0s, s1s, tmps = _schedule(block)
        for j in range(64):
            put_bits(SA.w(j, 0), wv[j])
        for i in range(48):
            put_limbs(SA.sched_sigma0(i, 0), s0s[i])
            put_limbs(SA.sched_sigma1(i, 0), s1s[i])
            put_limbs(SA.sched_tmp(i, 0), tmps[i])
        for j in range(4):
            put_bits(SA.a_chain(j, 0), h[:, 3 - j])
            put_bits(SA.e_chain(j, 0), h[:, 7 - j])

        def on_round(r, *vals):
            for fld, v in zip((SA.SIGMA1_E, SA.CH, SA.TMP1, SA.T1, SA.SIGMA0_A, SA.MAJ), vals[:6]):
                put_limbs(SA.rounds(r, fld, 0), v)
            put_bits(SA.a_chain(r + 4, 0), vals[6])
            put_bits(SA.e_chain(r + 4, 0), vals[7])
        fin = _rounds([h[:, j].copy() for j in range(8)], wv, on_round)
        for i in range(8):
            put_bits(SA.h_out(i, 0), h[:, i] + fin[i])
    return t


def output_words(fid, trace):
    """(n, 8) u32: the `h_out` bits of every row, packed."""
    one = (1 << 32) % _P[fid]
    bits = np.asarray(trace[:, SA.H_OUT:SA.H_OUT + 256], dtype=np.uint32).reshape(-1, 8, 32)
    assert np.all((bits == 0) | (bits == one))
    return ((bits == one).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


_DAGS = {}


def air_dag(field):
    """(nodes (n, 4) uint32, constraints) of Sha256Air over `field`."""
    if field.id not in _DAGS:
        air = SA.Sha256Air(field)
        _DAGS[field.id] = (air.nodes, air.constraints)
    return _DAGS[field.id]
