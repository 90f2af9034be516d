"""AIRs written with plonky3_b200.air's builder, shared by the constraint-program tests and tools/air_program_bench.py — test
infrastructure.

    fib_eval          uni-stark/tests/fib_air.rs:33-75 (2 columns, 3 public values)
    mul_air_eval      uni-stark/tests/mul_air.rs MulAir (20 repetitions x 3 columns, degree, boundary / transition switches)
"""
import numpy as np

REPETITIONS = 20


def fib_eval(b):
    m, pis = b.main(), b.public_values()
    l, r, nl, nr = m.local[0], m.local[1], m.next[0], m.next[1]
    b.when_first_row().assert_eq(l, pis[0])
    b.when_first_row().assert_eq(r, pis[1])
    t = b.when_transition()
    t.assert_eq(r, nl)
    t.assert_eq(l + r, nr)
    b.when_last_row().assert_eq(r, pis[2])


def fib_trace(field, n, a=0, b=1):
    rows = [(a, b)]
    for _ in range(n - 1):
        rows.append((rows[-1][1], (rows[-1][0] + rows[-1][1]) % field.P))
    return field.to_monty_array(np.array(rows, dtype=np.uint64)).astype(np.uint32)


def mul_air_eval(degree=3, boundary=True, transition=True):
    def ev(b):
        m = b.main()
        for i in range(REPETITIONS):
            a, bb, c = m.local[3 * i], m.local[3 * i + 1], m.local[3 * i + 2]
            b.assert_zero(a ** (degree - 1) * bb - c)
            if boundary:
                b.when_first_row().assert_eq(a * a + 1, bb)
            if transition:
                b.when_transition().assert_eq(a + REPETITIONS, m.next[3 * i])
    return ev


def mul_air_trace(field, rows, degree=3, boundary=True, transition=True, seed=1):
    """A valid MulAir trace (random_valid_trace's rules; numpy randomness instead of SmallRng)."""
    P = field.P
    rng = np.random.default_rng(seed)
    t = np.zeros((rows, 3 * REPETITIONS), dtype=np.int64)
    for r in range(rows):
        for i in range(REPETITIONS):
            k = r * REPETITIONS + i
            a = k % P if transition else int(rng.integers(0, P))
            b = (a * a + 1) % P if boundary and r == 0 else int(rng.integers(0, P))
            t[r, 3 * i], t[r, 3 * i + 1], t[r, 3 * i + 2] = a, b, pow(a, degree - 1, P) * b % P
    return field.to_monty_array(t.astype(np.uint64)).astype(np.uint32)

