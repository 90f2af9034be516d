"""AIRs written with plonky3_b200.air's builder, shared by the constraint-program tests and tools/air_program_bench.py — test
infrastructure.

    fib_eval          uni-stark/tests/fib_air.rs:33-75 (2 columns, 3 public values)
    mul_air_eval      uni-stark/tests/mul_air.rs MulAir (20 repetitions x 3 columns, degree, boundary / transition switches)
    poseidon2_eval    the vectorised Poseidon2 AIR of tools/quick_prove.py (KoalaBear width 16, degree-3 S-box, 4 + rounds_p + 4
                      rounds, VECTOR_LEN permutations per row), constraint for constraint as VectorizedPoseidon2Air's folder
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


def poseidon2_eval(field, constants, vector_len=8):
    """constants: uni_stark.RoundConstants (Montgomery)."""
    P = field.P
    beg = [[field.from_monty(int(v)) for v in r] for r in np.asarray(constants.beginning_full_round_constants).reshape(4, 16)]
    end = [[field.from_monty(int(v)) for v in r] for r in np.asarray(constants.ending_full_round_constants).reshape(4, 16)]
    part = [field.from_monty(int(v)) for v in np.asarray(constants.partial_round_constants).ravel()]
    rounds_p = len(part)
    ip = lambda k: pow(pow(2, k, P), P - 2, P)
    v16 = [P - 2, 1, 2, ip(1), 3, 4, P - ip(1), P - 3, P - 4, ip(8), ip(3), ip(24), P - ip(8), P - ip(3), P - ip(4), P - ip(24)]

    def mat4(x):
        a, b, c, d = x
        return [a * 2 + b * 3 + (c + d), a + b * 2 + (c * 3 + d), a + b + (c * 2 + d * 3), a * 3 + b + (c + d * 2)]

    def mds(s):
        s = sum((mat4(s[i:i + 4]) for i in range(0, 16, 4)), [])
        t = [s[k] + s[4 + k] + s[8 + k] + s[12 + k] for k in range(4)]
        return [s[i] + t[i % 4] for i in range(16)]

    cube = lambda x: x * x * x
    cols = 144 + rounds_p

    def ev(b):
        m = b.main()
        for v in range(vector_len):
            col = m.local[v * cols:(v + 1) * cols]
            s = mds(col[:16]); k = 16
            for rc in beg:
                s = mds([cube(s[i] + rc[i]) for i in range(16)])
                for i in range(16):
                    b.assert_eq(s[i], col[k + i]); s[i] = col[k + i]
                k += 16
            for r in range(rounds_p):
                b.assert_eq(cube(s[0] + part[r]), col[k]); s[0] = col[k]; k += 1
                t = s[0]
                for i in range(1, 16):
                    t = t + s[i]
                s = [s[i] * v16[i] + t for i in range(16)]
            for rc in end:
                s = mds([cube(s[i] + rc[i]) for i in range(16)])
                for i in range(16):
                    b.assert_eq(s[i], col[k + i]); s[i] = col[k + i]
                k += 16
    return ev, vector_len * cols
