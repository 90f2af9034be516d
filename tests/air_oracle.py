"""Oracle of the constraint-program quotient (p3gpu_air_quotient_dev) — test infrastructure.

Evaluates an AIR's node DAG (include/p3gpu.h p3gpu_air_node) directly over the quotient domain with the reference's formulas, in
vectorised int64 numpy on canonical integers; it never goes through the compiled program, so it is independent of the compiler:

    quotient domain   g * K, |K| = 2^log_q;  natural index i <-> memory row bitrev(i) of the committed bit-reversed LDE prefix
    next row          natural index (i + 2^q) mod |K|, q = log_q - log_n (vertically_packed_row wraps)
    selectors         selectors_on_coset (commit/src/domain.rs:321-361), unnormalised:
                      Z_H(x) = x^N - 1, first = Z_H / (x - 1), last = Z_H / (x - w_N^-1), transition = x - w_N^-1
    fold              sum_k c_k alpha^(K - 1 - k)  (decompose_alpha, air/src/symbolic/builder.rs:482-511)
    quotient          fold / Z_H(x)
"""
import numpy as np

CONST, MAIN_LOCAL, MAIN_NEXT, PUBLIC, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, ADD, SUB, NEG, MUL = range(11)

_PRIMES = {0: 0x78000001, 1: 0x7F000001}
_GEN = {0: 31, 1: 3}
_W = {0: 11, 1: 3}
_TOP = {0: (0x1A427A41, 27), 1: (0x6AC49F88, 24)}


def _root(fid, bits):
    top, adicity = _TOP[fid]
    return pow(top, 1 << (adicity - bits), _PRIMES[fid])


def _vpow(x, e, p):
    r = np.ones_like(x)
    b = x.copy()
    while e:
        if e & 1:
            r = r * b % p
        b = b * b % p
        e >>= 1
    return r


def _powers(w, n, p):
    """w^0 .. w^(n-1) as int64 (doubling)."""
    out = np.ones(n, dtype=np.int64)
    k = 1
    while k < n:
        out[k:2 * k] = out[:min(k, n - k)] * pow(w, k, p) % p
        k *= 2
    return out


def _bitrev(n_bits):
    i = np.arange(1 << n_bits, dtype=np.int64)
    r = np.zeros_like(i)
    for b in range(n_bits):
        r |= ((i >> b) & 1) << (n_bits - 1 - b)
    return r


def _ef_mul(a, b, p, w):
    r = [0] * 7
    for i in range(4):
        for j in range(4):
            r[i + j] += a[i] * b[j]
    return [(r[0] + w * r[4]) % p, (r[1] + w * r[5]) % p, (r[2] + w * r[6]) % p, r[3] % p]


def air_quotient(fid, nodes, constraints, lde_bitrev, log_q, log_n, public_values_monty, alpha_monty):
    """(2^log_q, 4) uint32 Montgomery quotient values in natural order.  lde_bitrev: the committed bit-reversed LDE (>= 2^log_q rows,
    Montgomery); public values and alpha: Montgomery words."""
    p = _PRIMES[fid]
    rinv = pow(1 << 32, p - 2, p)
    c = lambda m: int(m) * rinv % p
    nodes = np.asarray(nodes, dtype=np.int64).reshape(-1, 4)
    cons = [int(k) for k in np.asarray(constraints).ravel()]
    size, q = 1 << log_q, log_q - log_n
    lde = np.asarray(lde_bitrev, dtype=np.uint32)[:size].astype(np.int64)
    rows = _bitrev(log_q)
    nxt = (np.arange(size, dtype=np.int64) + (1 << q)) % size
    x = _GEN[fid] * _powers(_root(fid, log_q), size, p) % p
    zh = (_vpow(x, 1 << log_n, p) - 1) % p
    w_inv = pow(_root(fid, log_n), p - 2, p)
    selectors = {}

    def selector(op):
        if not selectors:
            selectors[IS_FIRST_ROW] = zh * _vpow((x - 1) % p, p - 2, p) % p
            selectors[IS_LAST_ROW] = zh * _vpow((x - w_inv) % p, p - 2, p) % p
            selectors[IS_TRANSITION] = (x - w_inv) % p
        return selectors[op]

    def column(col):
        return lde[rows, col] * rinv % p

    # reference counts, so a value is dropped after its last reader
    uses = np.zeros(len(nodes), dtype=np.int64)
    for op, a, b, _ in nodes:
        if op in (ADD, SUB, MUL):
            uses[a] += 1; uses[b] += 1
        elif op == NEG:
            uses[a] += 1
    for k in cons:
        uses[k] += 1
    vals = {}

    def take(i):
        v = vals[i]
        uses[i] -= 1
        if uses[i] == 0:
            del vals[i]
        return v

    for i, (op, a, b, imm) in enumerate(nodes):
        if uses[i] == 0:
            continue
        if op == CONST:
            v = np.int64(c(imm))
        elif op == MAIN_LOCAL:
            v = column(a)
        elif op == MAIN_NEXT:
            v = column(a)[nxt]
        elif op == PUBLIC:
            v = np.int64(c(public_values_monty[a]))
        elif op in (IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION):
            v = selector(op)
        elif op == ADD:
            v = (take(a) + take(b)) % p
        elif op == SUB:
            v = (take(a) - take(b)) % p
        elif op == NEG:
            v = (-take(a)) % p
        elif op == MUL:
            v = take(a) * take(b) % p
        else:
            raise ValueError(f"unknown op {op}")
        vals[i] = np.broadcast_to(np.asarray(v, dtype=np.int64), (size,)).copy() if np.ndim(v) == 0 else v
    alpha = [c(v) for v in alpha_monty]
    K = len(cons)
    apow = [[1, 0, 0, 0]]
    for _ in range(max(K - 1, 0)):
        apow.append(_ef_mul(apow[-1], alpha, p, _W[fid]))
    acc = np.zeros((size, 4), dtype=np.int64)
    for k, node in enumerate(cons):
        ck = take(node)
        for d in range(4):
            acc[:, d] = (acc[:, d] + ck * apow[K - 1 - k][d]) % p
    inv_zh = _vpow(zh, p - 2, p)
    out = acc * inv_zh[:, None] % p
    return ((out << 32) % p).astype(np.uint32)
