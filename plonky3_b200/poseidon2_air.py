"""The vectorised Poseidon2 permutation AIR (poseidon2-air/src): the AIR of `prove_prime_field_31 --objective
poseidon-2-permutations` (examples/src/airs.rs) over KoalaBear (the config-5 benchmark's statement) and BabyBear.

    air = VectorizedPoseidon2Air(KoalaBear, RoundConstants(beg, partial, end), gpu)
    trace = air.generate_trace_rows(inputs_dev)              # (n_perms, 16) int32 on the device -> (n_perms / 8, 1312)
    proof = uni_stark.prove(config, air, trace); uni_stark.verify(config, air, proof.to_postcard())

The two instances are the example's: KoalaBear has an x^3 S-box without registers and 20 partial rounds; BabyBear has an x^7
S-box with one register (the committed x^3, the S-box output is x3^2 x), 13 partial rounds, and a row of 8 x 298 = 2384 columns.

The constraints are written once, below, as a SymbolicAirBuilder eval in the order of poseidon2-air/src/air.rs; the verifier folds
them through SymbolicAir.eval_folded_constraints.  The prover does not use the constraint-program kernel: trace generation and the
quotient are the hand-written kernels of csrc/air.cu (p3gpu_p2air_generate_trace_dev / p3gpu_p2air_quotient_dev, and the
row-sharded p3gpu_p2air_quotient_sharded_dev that distributed.py runs), with no CPU fallback.

Column layout of one permutation (columns.rs): inputs [0,16) | 4 beginning full rounds {sbox registers [16 REG], post [16]} |
rounds_p partial rounds {sbox register [REG], post_sbox} | 4 ending full rounds {sbox registers, post}, REG = sbox_registers(field);
a row holds vector_len permutations side by side.  The row-sharded prove (distributed.prove_sharded) is KoalaBear-only for this AIR.  uni_stark re-exports RoundConstants, VectorizedPoseidon2Air and VECTOR_LEN.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .air import KernelAir
from .field import Field

VECTOR_LEN = 8           # examples/src/airs.rs: P2_VECTOR_LEN = 1 << 3


def sbox_registers(field) -> int:
    """SBOX_REGISTERS of the example's instance: BabyBear's x^7 S-box commits x^3 (1), KoalaBear's x^3 S-box commits nothing."""
    return 1 if field.SBOX_D == 7 else 0


def columns(field, rounds_p: int) -> int:
    """Columns of one permutation (columns.rs): 16 + 8 full rounds x 16 (REG + 1) + rounds_p (REG + 1)."""
    return 16 + (8 * 16 + rounds_p) * (sbox_registers(field) + 1)


@dataclass
class RoundConstants:
    """poseidon2-air/src/constants.rs:28-57 (Montgomery form)."""
    beginning_full_round_constants: np.ndarray    # (4, 16)
    partial_round_constants: np.ndarray           # (rounds_p,)
    ending_full_round_constants: np.ndarray       # (4, 16)


def poseidon2_eval(field, constants, vector_len=8):
    """(eval_fn, width) of VectorizedPoseidon2Air<.., WIDTH 16, SBOX_DEGREE, SBOX_REGISTERS, 4, rounds_p, vector_len>
    (poseidon2-air/src/air.rs eval) for the field's instance: KoalaBear (3, 0) with Poseidon2KoalaBear<16>'s internal diagonal
    (koala-bear/src/poseidon2.rs:410-428), BabyBear (7, 1) with Poseidon2BabyBear<16>'s (baby-bear/src/poseidon2.rs).  Per
    permutation: the committed post-state of every full round (16 each) and the S-box output of every partial round; with a
    register, each S-box's committed x^3 first (eval_sbox, case (7, 1): assert_eq(x3, x^3), output x3^2 x).
    constants: RoundConstants (Montgomery)."""
    P = field.P
    beg = [[field.from_monty(int(v)) for v in r] for r in np.asarray(constants.beginning_full_round_constants).reshape(4, 16)]
    end = [[field.from_monty(int(v)) for v in r] for r in np.asarray(constants.ending_full_round_constants).reshape(4, 16)]
    part = [field.from_monty(int(v)) for v in np.asarray(constants.partial_round_constants).ravel()]
    rounds_p = len(part)
    ip = lambda k: pow(pow(2, k, P), P - 2, P)
    reg = sbox_registers(field)
    if reg:
        v16 = [P - 2, 1, 2, ip(1), 3, 4, P - ip(1), P - 3, P - 4, ip(8), ip(2), ip(3), ip(27), P - ip(8), P - ip(4), P - ip(27)]
    else:
        v16 = [P - 2, 1, 2, ip(1), 3, 4, P - ip(1), P - 3, P - 4, ip(8), ip(3), ip(24), P - ip(8), P - ip(3), P - ip(4), P - ip(24)]

    def mat4(x):
        a, b, c, d = x
        return [a * 2 + b * 3 + (c + d), a + b * 2 + (c * 3 + d), a + b + (c * 2 + d * 3), a * 3 + b + (c + d * 2)]

    def mds(s):
        s = sum((mat4(s[i:i + 4]) for i in range(0, 16, 4)), [])
        t = [s[k] + s[4 + k] + s[8 + k] + s[12 + k] for k in range(4)]
        return [s[i] + t[i % 4] for i in range(16)]

    cube = lambda x: x * x * x
    cols = columns(field, rounds_p)

    def ev_registers(b, col):
        """The (7, 1) instance: every S-box checks its committed x^3 before its output is used."""
        s = mds(col[:16]); k = 16

        def full(s, k, rc):
            out = []
            for i in range(16):
                x = s[i] + rc[i]
                b.assert_eq(col[k + i], cube(x))
                out.append(col[k + i] * col[k + i] * x)
            s = mds(out); k += 16
            for i in range(16):
                b.assert_eq(s[i], col[k + i]); s[i] = col[k + i]
            return s, k + 16
        for rc in beg:
            s, k = full(s, k, rc)
        for r in range(rounds_p):
            x = s[0] + part[r]
            b.assert_eq(col[k], cube(x))
            b.assert_eq(col[k] * col[k] * x, col[k + 1]); s[0] = col[k + 1]; k += 2
            t = s[0]
            for i in range(1, 16):
                t = t + s[i]
            s = [s[i] * v16[i] + t for i in range(16)]
        for rc in end:
            s, k = full(s, k, rc)

    def ev(b):
        m = b.main()
        for v in range(vector_len):
            col = m.local[v * cols:(v + 1) * cols]
            if reg:
                ev_registers(b, col)
                continue
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


class VectorizedPoseidon2Air(KernelAir):
    """VectorizedPoseidon2Air<KoalaBear, ..., WIDTH 16, SBOX_DEGREE 3, SBOX_REGISTERS 0, 4, 20, VECTOR_LEN 8>, or the BabyBear
    instance <..., SBOX_DEGREE 7, SBOX_REGISTERS 1, 4, 13, ...>, in the surface uni_stark.prove and verify read: width
    vector_len * columns(field, rounds_p), max_constraint_degree 3 (the DAG's), no public values, and
    no transition constraints, so the next row is never opened (verifier.rs:431-440).  `gpu`: a plonky3_b200.gpu.Gpu (or None for a
    verifier-only AIR)."""
    air_name = "Poseidon2"

    def __init__(self, field: Field, constants: RoundConstants, gpu, vector_len: int = VECTOR_LEN):
        eval_fn, width = poseidon2_eval(field, constants, vector_len)
        super().__init__(field, width, eval_fn, main_next_row_columns=[], gpu=gpu)
        self.constants, self.vector_len = constants, vector_len
        self.rounds_p = int(np.asarray(constants.partial_round_constants).size)
        self._upload()

    def _upload(self):
        if self.gpu is None:
            return
        c = self.constants
        self.gpu.p2air_set_constants(self.field.id, c.beginning_full_round_constants, c.partial_round_constants, c.ending_full_round_constants)

    def generate_trace_rows(self, inputs_dev):
        """generate_vectorized_trace_rows (generation.rs:14-70): (n_perms, 16) device inputs -> (n_perms / 8, 8 columns) device
        trace (1312 columns for KoalaBear, 2384 for BabyBear)."""
        self._need_gpu("trace generation")
        self._upload()
        return self.gpu.p2air_generate_trace(self.field.id, inputs_dev, self.vector_len)

    def generate_trace_cols(self, inputs_dev, col0: int, col1: int):
        """Columns [col0, col1) of `generate_trace_rows(inputs_dev)` without building the full trace: one rank's column block
        for `distributed.prove_sharded` (KoalaBear only; the device refuses BabyBear)."""
        self._need_gpu("trace generation")
        self._upload()
        return self.gpu.p2air_generate_trace_cols(self.field.id, inputs_dev, int(col0), int(col1), self.vector_len)

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        """`trace_lde_dev`: the whole committed LDE.  Returns (its height, 4)."""
        self._upload()
        return self.gpu.p2air_quotient(self.field.id, trace_lde_dev, log_degree, alpha, self.vector_len)

    def _kernel_quotient_sharded(self, grp, log_lde_height: int, log_degree: int, alpha):
        """PeerGroup.p2air_quotient (KoalaBear only; the device refuses BabyBear)."""
        return grp.p2air_quotient(self.field, self.vector_len, log_lde_height, log_degree, alpha)
