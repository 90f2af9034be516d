"""Constraint-program AIRs for the row-sharded prove of SymbolicAirs, with valid traces — test infrastructure, shared by the
sharded-symbolic tests and tools/sharded_prove.py.

    wide_mul      a MulAir-style AIR of `width` columns: (width - 1) // 3 triples a^(d-1) b = c whose a steps by the triple count on
                  the next row, and counter columns (the rest) that step by one, the last of them 0 on the first row.  Degree d
                  (d = 3: two quotient chunks, log_blowup 1; d = 5: four, log_blowup 2); reads the next row in every 8-column unit.
    wide_fib      `width` / 2 Fibonacci pairs (fib_air.rs's constraints on every pair), pair 0 tied to 3 public values; degree
                  hint 3, so its quotient domain is the LDE domain at log_blowup 1.
    periodic      x_j steps by one on the next row, y_j = x_j p0 + p1 with periodic columns p0 (period 4) and p1 (period 8);
                  degree hint 3.
"""
import numpy as np

from plonky3_b200.air import SymbolicAir


def wide_mul_eval(width=64, degree=3):
    reps = (width - 1) // 3

    def ev(b):
        m = b.main()
        for i in range(reps):
            a, bb, c = m.local[3 * i], m.local[3 * i + 1], m.local[3 * i + 2]
            b.assert_zero(a ** (degree - 1) * bb - c)
            b.when_transition().assert_eq(a + reps, m.next[3 * i])
        for k in range(3 * reps, width):
            b.when_transition().assert_eq(m.local[k] + 1, m.next[k])
        b.when_first_row().assert_zero(m.local[width - 1])
    return ev


def wide_mul_trace(field, rows, width=64, degree=3, seed=1):
    P, reps = field.P, (width - 1) // 3
    rng = np.random.default_rng(seed)
    t = np.zeros((rows, width), dtype=np.int64)
    r = np.arange(rows, dtype=np.int64)
    for i in range(reps):
        a = (r * reps + i) % P
        bb = rng.integers(0, P, rows, dtype=np.int64)
        t[:, 3 * i], t[:, 3 * i + 1] = a, bb
        c = bb
        for _ in range(degree - 1):
            c = c * a % P                                   # < 2^62: exact in int64
        t[:, 3 * i + 2] = c
    for k in range(3 * reps, width):
        t[:, k] = (r + (0 if k == width - 1 else 7 * k)) % P
    return field.to_monty_array(t.astype(np.uint64)).astype(np.uint32)


def wide_mul(field, width=64, degree=3, gpu=None):
    return SymbolicAir(field, width, wide_mul_eval(width, degree), gpu=gpu)


def wide_fib_eval(width=32):
    def ev(b):
        m, pis = b.main(), b.public_values()
        for k in range(width // 2):
            l, r, nl, nr = m.local[2 * k], m.local[2 * k + 1], m.next[2 * k], m.next[2 * k + 1]
            t = b.when_transition()
            t.assert_eq(r, nl)
            t.assert_eq(l + r, nr)
        b.when_first_row().assert_eq(m.local[0], pis[0])
        b.when_first_row().assert_eq(m.local[1], pis[1])
        b.when_last_row().assert_eq(m.local[1], pis[2])
    return ev


def wide_fib_trace(field, rows, width=32):
    """Every pair k starts at (k, 1); returns (trace, public values of pair 0)."""
    P = field.P
    t = np.zeros((rows, width), dtype=np.int64)
    for k in range(width // 2):
        a, b = k, 1
        for r in range(rows):
            t[r, 2 * k], t[r, 2 * k + 1] = a, b
            a, b = b, (a + b) % P
    return field.to_monty_array(t.astype(np.uint64)).astype(np.uint32), [0, 1, int(t[rows - 1, 1])]


def wide_fib(field, width=32, gpu=None):
    return SymbolicAir(field, width, wide_fib_eval(width), num_public_values=3, max_constraint_degree=3, gpu=gpu)


P0, P1 = [1, 2, 3, 4], [5, 6, 7, 8, 9, 10, 11, 12]


def periodic_eval(width=32):
    def ev(b):
        m, (p0, p1) = b.main(), b.periodic_values()
        for j in range(width // 2):
            x, y = m.local[2 * j], m.local[2 * j + 1]
            b.assert_eq(y, x * p0 + p1)
            b.when_transition().assert_eq(x + 1, m.next[2 * j])
    return ev


def periodic_trace(field, rows, width=32):
    P = field.P
    t = np.zeros((rows, width), dtype=np.int64)
    r = np.arange(rows, dtype=np.int64)
    p0, p1 = np.array(P0)[r % len(P0)], np.array(P1)[r % len(P1)]
    for j in range(width // 2):
        x = (r + 3 * j) % P
        t[:, 2 * j], t[:, 2 * j + 1] = x, (x * p0 + p1) % P
    return field.to_monty_array(t.astype(np.uint64)).astype(np.uint32)


def periodic(field, width=32, gpu=None):
    return SymbolicAir(field, width, periodic_eval(width), max_constraint_degree=3, periodic_columns=[P0, P1], gpu=gpu)
