"""Oracle of the BabyBear Poseidon2 AIR (plonky3_b200.poseidon2_air, the (7, 1) instance) — test infrastructure, vectorised numpy
on canonical int64, written from the reference independently of `poseidon2_eval`:

    generation   poseidon2-air/src/generation.rs generate_trace_rows_for_perm with generate_sbox case (7, 1): one permutation ->
                 inputs[16] | 4 x {x3[16], post[16]} | rounds_p x {x3, post_sbox} | 4 x {x3[16], post[16]} (298 columns), a row
                 of vector_len permutations side by side (Montgomery words)
    constraints  poseidon2-air/src/air.rs eval, eval_full_round / eval_partial_round / eval_sbox case (7, 1): per full round the
                 16 checks x3 - x^3, then 16 checks mds_out - post; per partial round x3 - x^3, then x3^2 x - post_sbox
    quotient     the constraints folded with alpha^(K - 1 - k) over GENERATOR * K, |K| = the LDE height, divided by Z_H
                 (p3gpu_p2air_quotient_dev's contract)

The internal diagonal is the C oracle's Poseidon2BabyBear<16> diagonal (O.poseidon2_diag), not the one `poseidon2_eval` spells out.
"""
import numpy as np
import torch

import air_oracle as A
from oracle import p3_oracle as O
from plonky3_b200.field import BabyBear
from plonky3_b200.poseidon2_air import RoundConstants

F = BabyBear
P = F.P
ROUNDS_P = 13                        # Poseidon2BabyBear<16>'s partial rounds, the example's PARTIAL_ROUNDS
COLS = 16 + (8 * 16 + ROUNDS_P) * 2  # 298
CONSTRAINTS = (8 * 16 + ROUNDS_P) * 2  # 282


def constants_from_rng(rng) -> RoundConstants:
    """RoundConstants::from_rng (constants.rs): 4 x 16 beginning, 13 partial, 4 x 16 ending, drawn in that order (Montgomery)."""
    a = O.air_from_rng(F.id, rng, ROUNDS_P)
    return RoundConstants(np.array(a.beg, dtype=np.uint32).reshape(4, 16), np.array(a.part, dtype=np.uint32)[:ROUNDS_P],
                          np.array(a.end, dtype=np.uint32).reshape(4, 16))


def example_constants() -> RoundConstants:
    """The example binary's AIR constants: the first draws of SmallRng::seed_from_u64(1)."""
    return constants_from_rng(O.SmallRng(1))


def permutation(c: RoundConstants):
    """The C oracle's Poseidon2 permutation with the AIR's round constants (initial = beginning, terminal = ending)."""
    return O.make_perm(F.id, 16, np.asarray(c.beginning_full_round_constants).ravel(), np.asarray(c.ending_full_round_constants).ravel(),
                       np.asarray(c.partial_round_constants).ravel(), monty=True)


def _canon(c: RoundConstants):
    beg = F.from_monty_array(np.asarray(c.beginning_full_round_constants, dtype=np.uint32).reshape(4, 16)).astype(np.int64)
    part = F.from_monty_array(np.asarray(c.partial_round_constants, dtype=np.uint32).ravel()).astype(np.int64)
    end = F.from_monty_array(np.asarray(c.ending_full_round_constants, dtype=np.uint32).reshape(4, 16)).astype(np.int64)
    return beg, part, end


_DIAG = F.from_monty_array(O.poseidon2_diag(F.id, 16)).astype(np.int64)


def _mds_light(s):
    """external.rs: circ(2, 3, 1, 1) on each 4-block, then every element plus the sum of its position over the blocks."""
    out = np.empty_like(s)
    for b in range(0, 16, 4):
        x0, x1, x2, x3 = (s[:, b + i] for i in range(4))
        out[:, b] = (2 * x0 + 3 * x1 + x2 + x3) % P
        out[:, b + 1] = (x0 + 2 * x1 + 3 * x2 + x3) % P
        out[:, b + 2] = (x0 + x1 + 2 * x2 + 3 * x3) % P
        out[:, b + 3] = (3 * x0 + x1 + x2 + 2 * x3) % P
    sums = [(out[:, k] + out[:, 4 + k] + out[:, 8 + k] + out[:, 12 + k]) % P for k in range(4)]
    for i in range(16):
        out[:, i] = (out[:, i] + sums[i % 4]) % P
    return out


def _internal(s):
    total = s.sum(axis=1) % P
    return (s * _DIAG % P + total[:, None]) % P


def _cube(x):
    return x * x % P * x % P


def generate_perms(c: RoundConstants, inputs):
    """(n, 16) Montgomery inputs -> (n, 298) Montgomery: every permutation's columns."""
    beg, part, end = _canon(c)
    s = F.from_monty_array(np.ascontiguousarray(inputs, dtype=np.uint32).reshape(-1, 16)).astype(np.int64)
    parts = [s]
    s = _mds_light(s)

    def full(s, rc):
        x = (s + rc) % P
        x3 = _cube(x)
        parts.append(x3)
        s = _mds_light(x3 * x3 % P * x % P)
        parts.append(s)
        return s
    for rc in beg:
        s = full(s, rc)
    for r in range(len(part)):
        x = (s[:, 0] + part[r]) % P
        x3 = _cube(x)
        s = s.copy()
        s[:, 0] = x3 * x3 % P * x % P
        parts.append(np.stack([x3, s[:, 0]], axis=1))
        s = _internal(s)
    for rc in end:
        s = full(s, rc)
    t = np.concatenate(parts, axis=1)
    assert t.shape[1] == 16 + (8 * 16 + len(part)) * 2
    return F.to_monty_array(t)


def generate(c: RoundConstants, inputs, vector_len=8):
    """generate_vectorized_trace_rows: (n, 16) Montgomery inputs -> (n / vector_len, vector_len * 298) Montgomery trace."""
    x = np.ascontiguousarray(inputs, dtype=np.uint32).reshape(-1, 16)
    assert x.shape[0] % vector_len == 0
    return generate_perms(c, x).reshape(x.shape[0] // vector_len, -1)


def constraint_values_perms(c: RoundConstants, rows_canon):
    """(n, 298) canonical permutation columns -> (n, 282) canonical constraint values in air.rs's order."""
    beg, part, end = _canon(c)
    t = np.asarray(rows_canon, dtype=np.int64)
    out = []
    s = _mds_light(t[:, :16])
    k = 16

    def full(s, k, rc):
        x = (s + rc) % P
        reg = t[:, k:k + 16]
        out.append((reg - _cube(x)) % P)
        post = t[:, k + 16:k + 32]
        out.append((_mds_light(reg * reg % P * x % P) - post) % P)
        return post, k + 32
    for rc in beg:
        s, k = full(s, k, rc)
    for r in range(len(part)):
        x = (s[:, 0] + part[r]) % P
        reg, post = t[:, k], t[:, k + 1]
        out.append(((reg - _cube(x)) % P)[:, None])
        out.append(((reg * reg % P * x % P - post) % P)[:, None])
        s = s.copy()
        s[:, 0] = post
        s = _internal(s)
        k += 2
    for rc in end:
        s, k = full(s, k, rc)
    return np.concatenate(out, axis=1)


def constraint_values(c: RoundConstants, trace, vector_len=8):
    """(rows, vector_len * 298) Montgomery trace -> (rows, vector_len * 282) canonical constraint values."""
    t = F.from_monty_array(np.asarray(trace, dtype=np.uint32)).astype(np.int64)
    rows = t.shape[0]
    return constraint_values_perms(c, t.reshape(rows * vector_len, -1)).reshape(rows, -1)


def quotient(c: RoundConstants, lde_bitrev, log_n, alpha_monty, vector_len=8):
    """(H, 4) Montgomery quotient values in natural order over GENERATOR * K, |K| = H = the LDE height."""
    lde = np.asarray(lde_bitrev, dtype=np.uint32)
    H = lde.shape[0]
    log_h = H.bit_length() - 1
    vals = constraint_values(c, lde[A._bitrev(torch.arange(H), log_h).numpy()], vector_len)      # natural order
    K = vals.shape[1]
    alpha = [F.from_monty(int(v)) for v in alpha_monty]
    apow = [[1, 0, 0, 0]]
    for _ in range(K - 1):
        apow.append(A._ef_mul(apow[-1], alpha, P, F.EXT_W))
    coef = np.array(apow[::-1], dtype=np.int64)                                  # constraint k gets alpha^(K - 1 - k)
    acc = np.zeros((H, 4), dtype=np.int64)
    lo, hi = coef & 0xFFFF, coef >> 16                                          # 31 x 16-bit products: 2^47 each, sums < 2^59
    for d in range(4):
        acc[:, d] = ((vals @ lo[:, d]) % P + (vals @ hi[:, d]) % P * (1 << 16)) % P
    x = F.GENERATOR * A._powers(A._root(F.id, log_h), H, P, "cpu") % P
    zh = (A._vpow(x, 1 << log_n, P) - 1) % P
    out = acc * A._vpow(zh, P - 2, P).numpy()[:, None] % P
    return ((out << 32) % P).astype(np.uint32)
