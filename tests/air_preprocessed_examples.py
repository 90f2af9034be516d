"""AIRs with preprocessed and periodic columns, shared by the CPU and GPU tests of those columns — test infrastructure.

    mul_fib_pair     uni-stark/tests/mul_fib_pair.rs MulFibPAir: main (a, b), preprocessed (prod_coeff, sum_coeff) read on the
                     current row only (the next row is still opened: preprocessed_next_row_columns defaults to every column);
                     b' = prod_coeff * a * b + sum_coeff * (a + b), a' = b on transitions
    periodic_air     uni-stark/tests/periodic_air.rs PeriodicAir: main (x, y) equal to periodic columns of periods 4 and 2
    mixed            main (a, c), one preprocessed column s opened at zeta only (preprocessed_next_row_columns = []), periodic
                     columns u (period 4) and v (period 2): c = s * a * u (degree 3: two quotient chunks), a' = a + v on transitions

Each comes with a valid trace generator and, for tests/stark_verify_layout.py, its constraints written out by hand.
"""
import numpy as np

from plonky3_b200.air import SymbolicAir

PERIODIC_AIR_COLUMNS = [[1, 2, 3, 4], [10, 20]]
MIXED_PERIODIC = [[3, 1, 4, 1], [5, 9]]


def mul_fib_pair_preprocessed(field, n, tamper_index=None):
    rows = [[i % 2, (i + 1) % 6] for i in range(n)]
    if tamper_index is not None and tamper_index < n:
        rows[tamper_index][0] += 1
    return field.to_monty_array(np.array(rows, dtype=np.uint64)).astype(np.uint32)


def mul_fib_pair_eval(b):
    m, pre = b.main(), b.preprocessed()
    a, bb, na, nb = m.local[0], m.local[1], m.next[0], m.next[1]
    prod, s = pre.local[0], pre.local[1]
    t = b.when_transition()
    t.assert_eq(bb, na)
    t.assert_eq(prod * a * bb + s * (a + bb), nb)


def mul_fib_pair_air(field, n, gpu=None, tamper_index=None):
    return SymbolicAir(field, 2, mul_fib_pair_eval, gpu=gpu, preprocessed_trace=mul_fib_pair_preprocessed(field, n, tamper_index))


def mul_fib_pair_trace(field, n, a=0, b=1):
    P = field.P
    rows = [(a, b)]
    for i in range(1, n):
        pa, pb = rows[-1]
        prod, s = (i - 1) % 2, i % 6
        rows.append((pb, (prod * pa * pb + s * (pa + pb)) % P))
    return field.to_monty_array(np.array(rows, dtype=np.uint64)).astype(np.uint32)


def periodic_air_eval(b):
    m, p = b.main(), b.periodic_values()
    b.assert_eq(m.local[0], p[0])
    b.assert_eq(m.local[1], p[1])


def periodic_air(field, gpu=None, columns=None):
    return SymbolicAir(field, 2, periodic_air_eval, gpu=gpu, periodic_columns=columns or PERIODIC_AIR_COLUMNS)


def periodic_air_trace(field, n, columns=None):
    cols = columns or PERIODIC_AIR_COLUMNS
    rows = [[c[i % len(c)] for c in cols] for i in range(n)]
    return field.to_monty_array(np.array(rows, dtype=np.uint64)).astype(np.uint32)


def mixed_eval(b):
    m, pre, per = b.main(), b.preprocessed(), b.periodic_values()
    b.assert_eq(m.local[1], pre.local[0] * m.local[0] * per[0])
    b.when_transition().assert_eq(m.next[0], m.local[0] + per[1])


def mixed_preprocessed(field, n):
    return field.to_monty_array(np.array([[(7 * i + 2) % 11] for i in range(n)], dtype=np.uint64)).astype(np.uint32)


def mixed_air(field, n, gpu=None):
    return SymbolicAir(field, 2, mixed_eval, gpu=gpu, preprocessed_trace=mixed_preprocessed(field, n), preprocessed_next_row_columns=[],
                       periodic_columns=MIXED_PERIODIC)


def mixed_trace(field, n, a0=5):
    P = field.P
    u, v = MIXED_PERIODIC
    rows, a = [], a0
    for i in range(n):
        s = (7 * i + 2) % 11
        rows.append((a, s * a * u[i % 4] % P))
        a = (a + v[i % 2]) % P
    return field.to_monty_array(np.array(rows, dtype=np.uint64)).astype(np.uint32)


# ---- the same constraints for tests/stark_verify_layout.py (canonical EF lists, stark_verify's Fld arithmetic)
def _fold(f, cs, alpha):
    acc = [0, 0, 0, 0]
    for c in cs:
        acc = f.eadd(f.emul(acc, alpha), c)
    return acc


def stark_verify_air(name):
    if name == "mul_fib_pair":
        def constraints(f, loc, nxt, pis, first, last, trans, alpha, pre, pre_next, per):
            a, b = loc
            prod, s = pre
            c0 = f.emul(trans, f.esub(b, nxt[0]))
            c1 = f.emul(trans, f.esub(f.eadd(f.emul(f.emul(prod, a), b), f.emul(s, f.eadd(a, b))), nxt[1]))
            return _fold(f, [c0, c1], alpha)
        return {"width": 2, "main_next": True, "log_quotient_chunks": 1, "num_public_values": 0, "constraints": constraints,
                "preprocessed_width": 2, "preprocessed_next": True}
    if name == "periodic_air":
        def constraints(f, loc, nxt, pis, first, last, trans, alpha, pre, pre_next, per):
            return _fold(f, [f.esub(loc[0], per[0]), f.esub(loc[1], per[1])], alpha)
        return {"width": 2, "main_next": True, "log_quotient_chunks": 0, "num_public_values": 0, "constraints": constraints,
                "periodic": PERIODIC_AIR_COLUMNS}

    def constraints(f, loc, nxt, pis, first, last, trans, alpha, pre, pre_next, per):
        c0 = f.esub(loc[1], f.emul(f.emul(pre[0], loc[0]), per[0]))
        c1 = f.emul(trans, f.esub(nxt[0], f.eadd(loc[0], per[1])))
        return _fold(f, [c0, c1], alpha)
    return {"width": 2, "main_next": True, "log_quotient_chunks": 1, "num_public_values": 0, "constraints": constraints,
            "preprocessed_width": 1, "preprocessed_next": False, "periodic": MIXED_PERIODIC}
