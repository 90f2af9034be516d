"""Oracle of the constraint-program quotient for programs with preprocessed and periodic columns
(p3gpu_air_quotient_layout_dev) — test infrastructure, built on tests/air_oracle.py.

The new leaves become main-trace columns of an extended LDE prefix that tests/air_oracle.py evaluates unchanged:

    PREPROCESSED_LOCAL c / _NEXT c   MAIN_LOCAL / MAIN_NEXT of a column holding the preprocessed LDE's column c (memory row
                                     bitrev(i), next row bitrev(i + 2^q): read exactly as the trace)
    PERIODIC k                       MAIN_LOCAL of a column holding, at memory row bitrev(i), the periodic value of natural index i:
                                     P_k(x_i^(N / p_k)), P_k the degree < p_k interpolant of column k over the subgroup of size p_k,
                                     evaluated directly from its coefficients (not through the padded LDE table the prover builds);
                                     or, for a stand-in device, row i mod (table height) of a given table
"""
import numpy as np
import torch

import air_oracle as A

PREPROCESSED_LOCAL, PREPROCESSED_NEXT, PERIODIC = 16, 17, 18


def periodic_values(fid, column, log_q, log_n):
    """P(x_i^(N / p)) at every natural index i of the quotient domain g * K, |K| = 2^log_q (canonical int64): the interpolant's
    coefficients by a direct inverse DFT over the subgroup of size p = len(column), then Horner."""
    p = A._PRIMES[fid]
    col = np.asarray(column, dtype=np.int64) % p
    per = col.size
    x = (A._GEN[fid] * A._powers(A._root(fid, log_q), 1 << log_q, p, "cpu") % p).numpy()
    if per == 1:
        return np.full(x.shape, int(col[0]), dtype=np.int64)
    w_inv = pow(A._root(fid, per.bit_length() - 1), p - 2, p)
    n_inv = pow(per, p - 2, p)
    coeffs = []
    for k in range(per):                                               # c_k = (1/p) sum_j v_j w^(-jk)
        wk = A._powers(pow(w_inv, k, p), per, p, "cpu").tolist()
        coeffs.append(int(sum(int(v) * int(t) % p for v, t in zip(col, wk)) % p * n_inv % p))
    y = A._vpow(torch.from_numpy(x), (1 << log_n) // per, p).numpy()
    acc = np.zeros_like(x)
    for c in reversed(coeffs):
        acc = (acc * y + c) % p
    return acc


def air_quotient(fid, nodes, constraints, lde_bitrev, log_q, log_n, public_values_monty, alpha_monty, pre_lde_bitrev=None,
                 periodic_columns=None, periodic_table=None):
    """(2^log_q, 4) uint32 Montgomery quotient values in natural order, as air_oracle.air_quotient, with pre_lde_bitrev the committed
    bit-reversed preprocessed LDE (>= 2^log_q rows, Montgomery) and the periodic columns (canonical values) or a (rows, n_periodic)
    Montgomery periodic table."""
    p = A._PRIMES[fid]
    size = 1 << log_q
    lde = np.asarray(lde_bitrev, dtype=np.uint32)[:size]
    width = lde.shape[1]
    blocks = [lde]
    pre_width = 0
    if pre_lde_bitrev is not None:
        pre = np.asarray(pre_lde_bitrev, dtype=np.uint32)[:size]
        pre_width = pre.shape[1]
        blocks.append(pre)
    rows = A._bitrev(torch.arange(size, dtype=torch.int64), log_q).numpy()
    if periodic_table is not None:
        t = np.asarray(periodic_table, dtype=np.uint32)
        nat = t[np.arange(size) % t.shape[0]]
    elif periodic_columns:
        nat = np.stack([(periodic_values(fid, c, log_q, log_n) << 32) % p for c in periodic_columns], axis=1).astype(np.uint32)
    else:
        nat = np.zeros((size, 0), dtype=np.uint32)
    per = np.empty_like(nat)
    per[rows] = nat                                                    # natural index i at memory row bitrev(i)
    blocks.append(per)
    ext = np.ascontiguousarray(np.hstack(blocks))
    remapped = []
    for op, a, b, imm in np.asarray(nodes, dtype=np.int64).reshape(-1, 4).tolist():
        if op == PREPROCESSED_LOCAL:
            op, a = A.MAIN_LOCAL, width + a
        elif op == PREPROCESSED_NEXT:
            op, a = A.MAIN_NEXT, width + a
        elif op == PERIODIC:
            op, a = A.MAIN_LOCAL, width + pre_width + a
        remapped.append((op, a, b, imm))
    return A.air_quotient(fid, np.array(remapped, dtype=np.int64).reshape(-1, 4), constraints, ext, log_q, log_n, public_values_monty,
                          alpha_monty)
