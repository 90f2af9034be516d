"""The vectorised Poseidon1 permutation AIR (poseidon1-air/src): the AIR of `prove_prime_field_31 -o poseidon-1-permutations`
(examples/examples/prove_prime_field_31.rs), width 16, over BabyBear and KoalaBear.

    full, partial = Poseidon1Constants.from_fixture(KoalaBear, fixture).to_optimized()
    air = VectorizedPoseidon1Air(KoalaBear, (full, partial), gpu)
    trace = air.generate_trace_rows(inputs_dev)              # (n_perms, 16) int32 on the device -> (n_perms / 8, 8 * columns)
    proof = uni_stark.prove(config, air, trace); uni_stark.verify(config, air, proof.to_postcard())

The field fixes the S-box: KoalaBear x^3 without registers, BabyBear x^7 with one register (the committed x^3; the S-box output is
(x^3)^2 x).  The permutation runs in the optimized form of poseidon1/src/utils.rs: the partial rounds add one full constant
vector, apply the dense transition matrix m_i once, then per round the S-box on state[0], a scalar constant (none in the last
round) and a sparse matrix (first row `sparse_first_row[r]`, first column `v[r]`).  The committed values are those of that form.

Column layout of one permutation (columns.rs, repr(C)): inputs[16] | 4 x FullRound{sbox registers[16 * REG], post[16]} |
rounds_p x PartialRound{sbox registers[REG], post_sbox} | 4 x FullRound; a row holds vector_len permutations side by side, no
next-row reads, no selectors, no public values.

The constraints are written once, below, as a SymbolicAirBuilder eval in the order of poseidon1-air/src/air.rs; the verifier folds
them through SymbolicAir.eval_folded_constraints.  The prover runs the hand-written kernels of csrc/poseidon1_air.cu
(p3gpu_p1air_generate_trace_dev / p3gpu_p1air_quotient_dev), with no CPU fallback.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .air import KernelAir
from .field import Field

WIDTH, HALF_FULL_ROUNDS = 16, 4
VECTOR_LEN = 8           # examples/src/airs.rs: P2_VECTOR_LEN = 1 << 3, also the Poseidon1 objective's vector length


def sbox_registers(field: Field) -> int:
    """S-box registers of the reference example's instance: 1 for BabyBear (x^7), 0 for KoalaBear (x^3)."""
    return 1 if field.SBOX_D == 7 else 0


def columns(field: Field, rounds_p: int) -> int:
    """Columns of one permutation: 16 + 8 (16 REG + 16) + rounds_p (REG + 1)."""
    reg = sbox_registers(field)
    return WIDTH + 2 * HALF_FULL_ROUNDS * WIDTH * (reg + 1) + rounds_p * (reg + 1)


# ---------------------------------------------------------------- constants (canonical integers mod p)
def circulant(col, p):
    """circulant_to_dense (poseidon1/src/utils.rs): M[i][j] = col[(i - j) mod 16]."""
    n = len(col)
    return [[int(col[(i - j) % n]) % p for j in range(n)] for i in range(n)]


def _matmul(a, b, p):
    n = len(a)
    return [[sum(a[i][k] * b[k][j] for k in range(n)) % p for j in range(n)] for i in range(n)]


def _matvec(m, v, p):
    return [sum(mi * vi for mi, vi in zip(row, v)) % p for row in m]


def _transpose(m):
    return [list(r) for r in zip(*m)]


def _inverse(m, p):
    """Gauss-Jordan inverse over GF(p)."""
    n = len(m)
    aug = [list(r) + [int(i == j) for j in range(n)] for i, r in enumerate(m)]
    for c in range(n):
        piv = next(r for r in range(c, n) if aug[r][c] % p)
        aug[c], aug[piv] = aug[piv], aug[c]
        inv = pow(aug[c][c], p - 2, p)
        aug[c] = [x * inv % p for x in aug[c]]
        for r in range(n):
            if r != c and aug[r][c]:
                f = aug[r][c]
                aug[r] = [(x - f * y) % p for x, y in zip(aug[r], aug[c])]
    return [r[n:] for r in aug]


@dataclass
class FullRoundConstants:
    """poseidon1/src/external.rs FullRoundConstants (canonical): initial and terminal (4, 16) round constants; the dense MDS is the
    circulant of `mds_circ_col`."""
    initial: np.ndarray
    terminal: np.ndarray
    mds_circ_col: np.ndarray


@dataclass
class PartialRoundConstants:
    """poseidon1/src/internal.rs PartialRoundConstants (canonical): first_round_constants (16), m_i (16, 16), sparse_first_row
    (rounds_p, 16), v (rounds_p, 16; entry 15 is 0), round_constants (rounds_p - 1)."""
    first_round_constants: np.ndarray
    m_i: np.ndarray
    sparse_first_row: np.ndarray
    v: np.ndarray
    round_constants: np.ndarray

    @property
    def rounds_p(self) -> int:
        return int(np.asarray(self.sparse_first_row).shape[0])


@dataclass
class Poseidon1Constants:
    """poseidon1/src/lib.rs Poseidon1Constants, width 16, canonical: rounds_f full rounds split in halves, rounds_p partial rounds,
    the circulant MDS's first column, and rounds_f + rounds_p round-constant vectors (initial full | partial | terminal full)."""
    field: Field
    rounds_f: int
    rounds_p: int
    mds_circ_col: list
    round_constants: list

    @classmethod
    def from_fixture(cls, field: Field, entry: dict) -> "Poseidon1Constants":
        """One field's entry of tests/golden/poseidon1_constants.json (tools/gen_constants.py)."""
        return cls(field, int(entry["rounds_f"]), int(entry["rounds_p"]), [int(v) for v in entry["mds_circ_col"]],
                   [[int(v) for v in r] for r in entry["round_constants"]])

    def dense_mds(self):
        return circulant(self.mds_circ_col, self.field.P)

    def to_optimized(self):
        """Poseidon1Constants::to_optimized (poseidon1/src/lib.rs, utils.rs compute_optimized_constants): the sparse
        decomposition of the MDS (working on M^T, HorizenLabs' order, reversed) and the round-constant compression by backward
        substitution through M^-1.  Returns (FullRoundConstants, PartialRoundConstants)."""
        p, n, half, rp = self.field.P, WIDTH, self.rounds_f // 2, self.rounds_p
        assert len(self.round_constants) == self.rounds_f + rp and rp >= 1
        rc = [[int(v) % p for v in r] for r in self.round_constants]
        initial, partial, terminal = rc[:half], rc[half:half + rp], rc[half + rp:]
        mds = self.dense_mds()
        # equivalent_round_constants
        mds_inv = _inverse(mds, p)
        opt = [0] * rp
        tmp = list(partial[rp - 1])
        for i in range(rp - 2, -1, -1):
            inv_cip = _matvec(mds_inv, tmp, p)
            opt[i + 1] = inv_cip[0]
            tmp = [partial[i][0]] + [(partial[i][j] + inv_cip[j]) % p for j in range(1, n)]
        first_rc = tmp
        # compute_equivalent_matrices
        mds_t = _transpose(mds)
        m_mul, m_i = mds_t, None
        vs, ws = [], []
        for _ in range(rp):
            vs.append([m_mul[0][j + 1] for j in range(n - 1)] + [0])
            w = [m_mul[i][0] for i in range(1, n)]
            m_hat_inv = _inverse([r[1:] for r in m_mul[1:]], p)
            ws.append([sum(a * b for a, b in zip(m_hat_inv[i], w)) % p for i in range(n - 1)] + [0])
            m_i = [list(r) for r in m_mul]
            m_i[0] = [1] + [0] * (n - 1)
            for r in m_i[1:]:
                r[0] = 0
            m_mul = _matmul(mds_t, m_i, p)
        m_i = _transpose(m_i)
        vs.reverse(); ws.reverse()
        first_rows = [[mds[0][0]] + w[:n - 1] for w in ws]
        a = lambda x: np.array(x, dtype=np.int64)
        return (FullRoundConstants(a(initial), a(terminal), a([int(c) % p for c in self.mds_circ_col])),
                PartialRoundConstants(a(first_rc), a(m_i), a(first_rows), a(vs), a(opt[1:])))


# ---------------------------------------------------------------- constraints
def poseidon1_eval(field: Field, full: FullRoundConstants, partial: PartialRoundConstants, vector_len: int = VECTOR_LEN):
    """(eval_fn, width) of VectorizedPoseidon1Air<F, WIDTH 16, SBOX_DEGREE, SBOX_REGISTERS, 4, rounds_p, vector_len>
    (poseidon1-air/src/air.rs eval, vectorized.rs): permutation 0's constraints, then permutation 1's, and so on.  Per full round
    the 16 register checks x3 - x^3 (BabyBear), then the 16 post checks mds_out - post; per partial round the register check
    (BabyBear), then sbox_out - post_sbox.  Constants canonical."""
    reg = sbox_registers(field)
    rp = partial.rounds_p
    cols = columns(field, rp)
    ini = [[int(v) for v in r] for r in np.asarray(full.initial).reshape(HALF_FULL_ROUNDS, WIDTH)]
    ter = [[int(v) for v in r] for r in np.asarray(full.terminal).reshape(HALF_FULL_ROUNDS, WIDTH)]
    circ = [int(v) for v in np.asarray(full.mds_circ_col).ravel()]
    frc = [int(v) for v in np.asarray(partial.first_round_constants).ravel()]
    m_i = [[int(v) for v in r] for r in np.asarray(partial.m_i).reshape(WIDTH, WIDTH)]
    sfr = [[int(v) for v in r] for r in np.asarray(partial.sparse_first_row).reshape(rp, WIDTH)]
    vv = [[int(v) for v in r] for r in np.asarray(partial.v).reshape(rp, WIDTH)]
    prc = [int(v) for v in np.asarray(partial.round_constants).ravel()]

    def sbox(b, x, regs):
        if reg == 0:
            return x * x * x
        b.assert_eq(regs[0], x * x * x)
        return regs[0] * regs[0] * x

    def mds(s):
        return [sum((s[j] * circ[(i - j) % WIDTH] for j in range(1, WIDTH)), s[0] * circ[i]) for i in range(WIDTH)]

    def ev(b):
        m = b.main()
        for v in range(vector_len):
            col = m.local[v * cols:(v + 1) * cols]
            s, k = list(col[:WIDTH]), WIDTH

            def full_round(s, k, rc):
                regs, post = col[k:k + WIDTH * reg], col[k + WIDTH * reg:k + WIDTH * (reg + 1)]
                s = [sbox(b, s[i] + rc[i], regs[i:i + 1]) for i in range(WIDTH)]
                s = mds(s)
                for i in range(WIDTH):
                    b.assert_eq(s[i], post[i])
                return list(post), k + WIDTH * (reg + 1)
            for rc in ini:
                s, k = full_round(s, k, rc)
            s = [s[i] + frc[i] for i in range(WIDTH)]
            s = [sum((s[j] * m_i[i][j] for j in range(1, WIDTH)), s[0] * m_i[i][0]) for i in range(WIDTH)]
            for r in range(rp):
                out = sbox(b, s[0], col[k:k + reg])
                post = col[k + reg]
                b.assert_eq(out, post)
                k += reg + 1
                s0 = post + prc[r] if r < rp - 1 else post
                new0 = sum((s[j] * sfr[r][j] for j in range(1, WIDTH)), s0 * sfr[r][0])
                s = [new0] + [s[i] + s0 * vv[r][i - 1] for i in range(1, WIDTH)]
            for rc in ter:
                s, k = full_round(s, k, rc)
            assert k == cols
    return ev, vector_len * cols


# ---------------------------------------------------------------- inputs
def random_inputs(field: Field, n: int, seed: int = 1) -> np.ndarray:
    """(n, 16) uint32 Montgomery words: `SmallRng::seed_from_u64(seed)` then `rng.random::<[F; 16]>()` n times
    (poseidon1-air/src/vectorized.rs:231-232), MontyField31's rejection-sampled draw.

    rand's SmallRng is xoshiro256++ seeded through SplitMix64 (keccak_air.random_inputs); a field element takes `next_u32` (the
    high half of one `next_u64`) shifted right by one, redrawn while >= p, and that value is the Montgomery representation
    itself.  A scalar restatement in Python: slow for millions of permutations."""
    M = (1 << 64) - 1
    s, x = [], seed & M
    for _ in range(4):
        x = (x + 0x9E3779B97F4A7C15) & M
        z = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        s.append(z ^ (z >> 31))
    s0, s1, s2, s3 = s
    P, out, k = field.P, np.empty(16 * n, dtype=np.uint32), 0
    while k < out.size:
        t = (s0 + s3) & M
        v = ((((t << 23) | (t >> 41)) + s0) & M) >> 33
        t = (s1 << 17) & M
        s2 ^= s0; s3 ^= s1; s1 ^= s2; s0 ^= s3; s2 ^= t
        s3 = ((s3 << 45) | (s3 >> 19)) & M
        if v < P:
            out[k] = v
            k += 1
    return out.reshape(n, 16)


class VectorizedPoseidon1Air(KernelAir):
    """VectorizedPoseidon1Air<F, WIDTH 16, SBOX_DEGREE, SBOX_REGISTERS, 4, rounds_p, VECTOR_LEN 8> in the surface uni_stark.prove
    and verify read: width vector_len * columns(field, rounds_p), max_constraint_degree 3, no public values, no next-row opening.
    `constants`: (FullRoundConstants, PartialRoundConstants) as Poseidon1Constants.to_optimized returns them.  `gpu`: a
    plonky3_b200.gpu.Gpu (or None for a verifier-only AIR)."""
    air_name = "Poseidon1"

    def __init__(self, field: Field, constants, gpu=None, vector_len: int = VECTOR_LEN):
        full, partial = constants
        eval_fn, width = poseidon1_eval(field, full, partial, vector_len)
        super().__init__(field, width, eval_fn, main_next_row_columns=[], max_constraint_degree=3, gpu=gpu)
        self.full, self.partial, self.vector_len = full, partial, vector_len
        self.rounds_p = partial.rounds_p
        self._upload()

    def _upload(self):
        if self.gpu is None:
            return
        f, full, part = self.field, self.full, self.partial
        mo = lambda a: f.to_monty_array(np.asarray(a, dtype=np.int64) % f.P)
        self.gpu.p1air_set_constants(f.id, mo(full.initial), mo(full.terminal), mo(full.mds_circ_col), mo(part.first_round_constants),
                                     mo(part.m_i), mo(part.round_constants), mo(part.sparse_first_row), mo(part.v), part.rounds_p)

    def generate_trace_rows(self, inputs_dev):
        """generate_vectorized_trace_rows (poseidon1-air/src/generation.rs): (n_perms, 16) device Montgomery inputs, n_perms
        vector_len times a power of two -> the (n_perms / vector_len, width) device trace."""
        self._need_gpu("trace generation")
        self._upload()
        return self.gpu.p1air_generate_trace(self.field.id, inputs_dev, self.vector_len)

    def generate_trace_cols(self, inputs_dev, col0: int, col1: int):
        """Columns [col0, col1) of `generate_trace_rows(inputs_dev)` without building the full trace: one rank's column block for
        `distributed.prove_sharded`.  The window may cut a permutation."""
        self._need_gpu("trace generation")
        self._upload()
        return self.gpu.p1air_generate_trace_cols(self.field.id, inputs_dev, int(col0), int(col1), self.vector_len)

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        """`trace_lde_dev`: the trace on GENERATOR * K, |K| = 2N (the committed LDE's prefix).  Returns (2N, 4)."""
        self._upload()
        return self.gpu.p1air_quotient(self.field.id, trace_lde_dev, int(log_degree), alpha, self.vector_len)

    def _kernel_quotient_sharded(self, grp, log_lde_height: int, log_degree: int, alpha):
        self._upload()
        return self.gpu.p1air_quotient_sharded(self.field.id, grp.struct, grp.col_starts, log_lde_height, log_degree, alpha, self.vector_len)
