"""Oracle of the Keccak-f AIR (plonky3_b200.keccak_air) — test infrastructure.

    generate(fid, inputs)        generate_trace_rows (keccak-air/src/generation.rs:16-161) restated in numpy, vectorised over the
                                 permutations: (H, 2633) Montgomery words, padding included.  The round function follows FIPS 202
                                 (theta, rho + pi, chi, iota) on the state words; the trace columns are the generation.rs values.
    constraint_values(...)       the AIR's constraint DAG evaluated on every row of a trace with check_constraints' semantics
                                 (air/src/check_constraints.rs: next row i + 1 mod H, is_first_row = [i = 0], is_last_row =
                                 [i = H - 1], is_transition = 1 - is_last_row): (n_constraints, H) canonical values.
    air_dag(field)               the AIR's (nodes, constraints), built once per field.
"""
import numpy as np

from plonky3_b200 import keccak_air as KA

CONST, MAIN_LOCAL, MAIN_NEXT, PUBLIC, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, ADD, SUB, NEG, MUL = range(11)
_P = {0: 0x78000001, 1: 0x7F000001}
_U = np.uint64


def _rotl(v, r):
    return v if r == 0 else (v << _U(r)) | (v >> _U(64 - r))


def _bits(fid, w):
    """(..., 64) Montgomery 0 / 1 of the bits of u64 words, least significant first."""
    one = (1 << 32) % _P[fid]
    return (((w[..., None] >> np.arange(64, dtype=np.uint64)) & _U(1)) * _U(one)).astype(np.uint32)


def _limbs(fid, w):
    """(..., 4) Montgomery 16-bit limbs of u64 words, least significant first."""
    one = (1 << 32) % _P[fid]
    v = (w[..., None] >> (np.arange(4, dtype=np.uint64) * _U(16))) & _U(0xFFFF)
    return (v * _U(one) % _U(_P[fid])).astype(np.uint32)


def perm_rows(fid, inputs):
    """(n, 25) u64 inputs (input[x + 5 y] = state[x][y]) -> (n, 24, 2633): the 24 rows of each permutation."""
    inputs = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(-1, 25)
    n = inputs.shape[0]
    one = (1 << 32) % _P[fid]
    out = np.zeros((n, KA.NUM_ROUNDS, KA.WIDTH), dtype=np.uint32)
    st = inputs.copy()                                                     # st[:, x + 5 y] = A[x][y]
    pre = _limbs(fid, inputs).reshape(n, 100)                              # preimage[y][x][limb]: (5 y + x) * 4 + limb
    for r in range(KA.NUM_ROUNDS):
        row = out[:, r]
        row[:, KA.STEP_FLAGS + r] = one
        row[:, KA.PREIMAGE:KA.A] = pre
        row[:, KA.A:KA.C] = _limbs(fid, st).reshape(n, 100)
        c = st[:, 0:5] ^ st[:, 5:10] ^ st[:, 10:15] ^ st[:, 15:20] ^ st[:, 20:25]
        cp = c ^ np.roll(c, 1, axis=1) ^ _rotl(np.roll(c, -1, axis=1), 1)  # C[x] ^ C[x - 1] ^ ROT(C[x + 1], 1)
        ap = st ^ np.tile(c ^ cp, 5)                                        # A' = A ^ C ^ C'
        row[:, KA.C:KA.C_PRIME] = _bits(fid, c).reshape(n, 320)
        row[:, KA.C_PRIME:KA.A_PRIME] = _bits(fid, cp).reshape(n, 320)
        row[:, KA.A_PRIME:KA.A_PRIME_PRIME] = _bits(fid, ap).reshape(n, 1600)
        # pi + rho: B[y][(2x + 3y) % 5] = ROT(A'[x][y], R[x][y]); chi: A''[x][y] = B[x][y] ^ (~B[x+1][y] & B[x+2][y])
        bb = np.zeros_like(st)
        for x in range(5):
            for y in range(5):
                bb[:, y + 5 * ((2 * x + 3 * y) % 5)] = _rotl(ap[:, x + 5 * y], KA.R[x][y])
        app = np.empty_like(st)
        for x in range(5):
            for y in range(5):
                app[:, x + 5 * y] = bb[:, x + 5 * y] ^ (~bb[:, (x + 1) % 5 + 5 * y] & bb[:, (x + 2) % 5 + 5 * y])
        row[:, KA.A_PRIME_PRIME:KA.A_PRIME_PRIME_0_0_BITS] = _limbs(fid, app).reshape(n, 100)
        row[:, KA.A_PRIME_PRIME_0_0_BITS:KA.A_PRIME_PRIME_PRIME_0_0_LIMBS] = _bits(fid, app[:, 0])
        st = app
        st[:, 0] ^= _U(KA.RC[r])                                            # iota
        row[:, KA.A_PRIME_PRIME_PRIME_0_0_LIMBS:] = _limbs(fid, st[:, 0])
    return out


def height(n):
    return 1 << max(24 * n - 1, 0).bit_length()


def generate(fid, inputs):
    """The full trace: the permutations' rows, then the zero-input permutation's rows repeated up to the power-of-two height."""
    inputs = np.asarray(inputs, dtype=np.uint64).reshape(-1, 25)
    n = inputs.shape[0]
    H = height(n)
    real = perm_rows(fid, inputs).reshape(24 * n, KA.WIDTH)
    zero = perm_rows(fid, np.zeros((1, 25), dtype=np.uint64))[0]
    pad = np.tile(zero, (-(-(H - 24 * n) // 24), 1))[: H - 24 * n]
    return np.concatenate([real, pad]) if n else pad


def output_state(fid, trace, perm):
    """The u64 state a''' of row 24 perm + 23, input-indexed (x + 5 y)."""
    p = _P[fid]
    rinv = pow(1 << 32, p - 2, p)
    row = trace[24 * perm + 23].astype(np.int64)
    canon = lambda col: int(row[col]) * rinv % p
    out = np.zeros(25, dtype=np.uint64)
    for y in range(5):
        for x in range(5):
            out[x + 5 * y] = sum(canon(KA.a_prime_prime_prime(y, x, l)) << (16 * l) for l in range(4))
    return out


_DAGS = {}


def air_dag(field):
    """(nodes (n, 4) uint32, constraints) of KeccakAir over `field`."""
    if field.id not in _DAGS:
        air = KA.KeccakAir(field)
        _DAGS[field.id] = (air.nodes, air.constraints)
    return _DAGS[field.id]


def constraint_values(fid, nodes, constraints, trace):
    """(K, H) int64: constraint k at row i of the Montgomery trace, canonical."""
    p = _P[fid]
    rinv = pow(1 << 32, p - 2, p)
    t = np.asarray(trace, dtype=np.uint32).astype(np.int64) * rinv % p
    H = t.shape[0]
    first = np.zeros(H, dtype=np.int64); first[0] = 1
    last = np.zeros(H, dtype=np.int64); last[-1] = 1
    sel = {IS_FIRST_ROW: first, IS_LAST_ROW: last, IS_TRANSITION: 1 - last}
    vals = []
    for op, a, b, imm in np.asarray(nodes, dtype=np.int64):
        if op == CONST:
            v = np.full(H, int(imm) * rinv % p, dtype=np.int64)
        elif op == MAIN_LOCAL:
            v = t[:, a]
        elif op == MAIN_NEXT:
            v = np.roll(t[:, a], -1)
        elif op in sel:
            v = sel[op]
        elif op == ADD:
            v = (vals[a] + vals[b]) % p
        elif op == SUB:
            v = (vals[a] - vals[b]) % p
        elif op == NEG:
            v = (-vals[a]) % p
        elif op == MUL:
            v = vals[a] * vals[b] % p
        else:
            raise ValueError(f"unexpected op {op}")
        vals.append(v)
    return np.stack([vals[int(k)] for k in constraints])
