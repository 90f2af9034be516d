"""The Blake3 compression AIR (blake3-air/src): the AIR of `prove_prime_field_31 --objective blake-3-permutations`
(examples/src/airs.rs), over BabyBear and KoalaBear.

    air = Blake3Air(KoalaBear, gpu)
    trace = air.generate_random_trace_rows(1 << 18)           # or air.generate_trace_rows(inputs_dev), (n, 24) int32 on the device
    proof = uni_stark.prove(config, air, trace); uni_stark.verify(config, air, proof.to_postcard())

One row per compression, rows independent: no selectors, no next-row reads, no public values.  The constraints are written once,
below, as a SymbolicAirBuilder eval that follows blake3-air/src/air.rs and air/src/utils.rs line by line; the verifier folds them
through SymbolicAir.eval_folded_constraints.  The prover does not use the constraint-program kernel (9632 constraints are past its
limit): trace generation and the quotient are the hand-written kernels of csrc/blake3_air.cu (p3gpu_blake3_air_generate_trace_dev
/ p3gpu_blake3_air_quotient_dev), with no CPU fallback.

Column layout (columns.rs Blake3Cols, repr(C)): inputs [16][32] bits [0,512) | chaining_values [2][4][32] [512,768) |
counter_low, counter_hi, block_len, flags (32 bits each) [768,896) | initial_row0 [4][2] limbs [896,904) | initial_row2 [904,912) |
7 FullRounds [912,8528) | final_round_helpers [4][32] [8528,8656) | outputs [4][4][32] [8656,9168).  A FullRound is four
Blake3States (state_prime, state_middle, state_middle_prime, state_output); a Blake3State is 272 columns: row0 [4][2] 16-bit limbs,
row1 [4][32] bits, row2 [4][2] limbs, row3 [4][32] bits.  Bits are least significant first, limbs [lo, hi].
"""
from __future__ import annotations

import numpy as np

from .air import KernelAir
from .field import Field

WIDTH = 9168
NUM_ROUNDS, BITS_PER_LIMB = 7, 16
INPUTS, CHAINING_VALUES, COUNTER_LOW, COUNTER_HI, BLOCK_LEN, FLAGS = 0, 512, 768, 800, 832, 864
INITIAL_ROW0, INITIAL_ROW2, FULL_ROUNDS, FINAL_ROUND_HELPERS, OUTPUTS = 896, 904, 912, 8528, 8656
STATE_WIDTH, FULL_ROUND_WIDTH = 272, 4 * 272
STATE_PRIME, STATE_MIDDLE, STATE_MIDDLE_PRIME, STATE_OUTPUT = 0, 1, 2, 3      # a FullRound's states, in column order

IV = [0x6A09E667, 0xBB67AE85, 0x3C6EF372, 0xA54FF53A, 0x510E527F, 0x9B05688C, 0x1F83D9AB, 0x5BE0CD19]   # constants.rs, as u32
MSG_PERMUTATION = [2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8]


# Blake3Cols column indices (columns.rs)
def inputs(w, i): return INPUTS + 32 * w + i
def chaining_values(h, j, i): return CHAINING_VALUES + 128 * h + 32 * j + i
def initial_row0(j, limb): return INITIAL_ROW0 + 2 * j + limb
def initial_row2(j, limb): return INITIAL_ROW2 + 2 * j + limb
def state(r, s): return FULL_ROUNDS + FULL_ROUND_WIDTH * r + STATE_WIDTH * s          # first column of full_rounds[r]'s state s
def row0(base, j, limb): return base + 2 * j + limb
def row1(base, j, i): return base + 8 + 32 * j + i
def row2(base, j, limb): return base + 136 + 2 * j + limb
def row3(base, j, i): return base + 144 + 32 * j + i
def final_round_helpers(j, i): return FINAL_ROUND_HELPERS + 32 * j + i
def outputs(o, j, i): return OUTPUTS + 128 * o + 32 * j + i


def _xor(p, q): return p + q - p * (2 * q)           # PrimeCharacteristicRing::xor: x + y - x * 2y


def pack_bits_le(bits):
    """air/src/utils.rs pack_bits_le: bits.rev().reduce(|acc, b| acc.double() + b), least significant first."""
    acc = None
    for v in reversed(bits):
        acc = v if acc is None else acc * 2 + v
    return acc


def add3(bld, a, b, c, d):
    """air/src/utils.rs add3: a = b + c + d mod 2^32 on [lo, hi] 16-bit limbs; two constraints."""
    two_16, two_32 = 1 << 16, 1 << 32
    acc_16 = a[0] - b[0] - c[0] - d[0]
    acc_32 = a[1] - b[1] - c[1] - d[1]
    acc = acc_16 + acc_32 * two_16
    bld.assert_zero(acc * (acc + two_32) * (acc + 2 * two_32))
    bld.assert_zero(acc_16 * (acc_16 + two_16) * (acc_16 + 2 * two_16))


def add2(bld, a, b, c):
    """air/src/utils.rs add2: a = b + c mod 2^32 on [lo, hi] 16-bit limbs; two constraints."""
    two_16, two_32 = 1 << 16, 1 << 32
    acc_16 = a[0] - b[0] - c[0]
    acc_32 = a[1] - b[1] - c[1]
    acc = acc_16 + acc_32 * two_16
    bld.assert_zero(acc * (acc + two_32))
    bld.assert_zero(acc_16 * (acc_16 + two_16))


def xor_32_shift(bld, a, b, c, shift):
    """air/src/utils.rs xor_32_shift: a = b ^ (c << shift) with a as [lo, hi] limbs, b and c as 32 bits; 32 booleans of c, then
    the two limbs."""
    for v in c:
        bld.assert_bool(v)
    lo = pack_bits_le([_xor(b[i], c[(32 + i - shift) % 32]) for i in range(16)])
    hi = pack_bits_le([_xor(b[i + 16], c[(32 + i + 16 - shift) % 32]) for i in range(16)])
    bld.assert_zero(a[0] - lo)
    bld.assert_zero(a[1] - hi)


class _State:
    """A Blake3State of expressions: row0 / row2 as four [lo, hi] limb pairs, row1 / row3 as four 32-bit lists."""

    def __init__(self, r0, r1, r2, r3):
        self.row0, self.row1, self.row2, self.row3 = r0, r1, r2, r3


def _trace_state(local, base):
    return _State([[local[row0(base, j, l)] for l in range(2)] for j in range(4)],
                  [[local[row1(base, j, i)] for i in range(32)] for j in range(4)],
                  [[local[row2(base, j, l)] for l in range(2)] for j in range(4)],
                  [[local[row3(base, j, i)] for i in range(32)] for j in range(4)])


def _quarter_round(bld, a, b, c, d, m0, a1, b1, c1, d1, m1, a2, b2, c2, d2):
    """Blake3Air::quarter_round_function (air.rs:43-111): inputs a b c d, half-way values a1 .. d1, outputs a2 .. d2."""
    add3(bld, a1, a, [pack_bits_le(b[:16]), pack_bits_le(b[16:])], m0)
    xor_32_shift(bld, a1, d, d1, 16)
    add2(bld, c1, c, [pack_bits_le(d1[:16]), pack_bits_le(d1[16:])])
    xor_32_shift(bld, c1, b, b1, 12)
    add3(bld, a2, a1, [pack_bits_le(b1[:16]), pack_bits_le(b1[16:])], m1)
    xor_32_shift(bld, a2, d1, d2, 8)
    add2(bld, c2, c1, [pack_bits_le(d2[:16]), pack_bits_le(d2[16:])])
    xor_32_shift(bld, c2, b1, b2, 7)


def _verify_round(bld, inp, rnd, m):
    """Blake3Air::verify_round (air.rs:175-229): the four column quarter rounds, then the four diagonal ones."""
    sp, sm, smp, so = rnd
    for i in range(4):
        _quarter_round(bld, inp.row0[i], inp.row1[i], inp.row2[i], inp.row3[i], m[2 * i],
                       sp.row0[i], sp.row1[i], sp.row2[i], sp.row3[i], m[2 * i + 1],
                       sm.row0[i], sm.row1[i], sm.row2[i], sm.row3[i])
    for i in range(4):
        j1, j2, j3 = (i + 1) % 4, (i + 2) % 4, (i + 3) % 4
        _quarter_round(bld, sm.row0[i], sm.row1[j1], sm.row2[j2], sm.row3[j3], m[2 * i + 8],
                       smp.row0[i], smp.row1[j1], smp.row2[j2], smp.row3[j3], m[2 * i + 9],
                       so.row0[i], so.row1[j1], so.row2[j2], so.row3[j3])


def eval_blake3(bld):
    """Air::eval for Blake3Air (blake3-air/src/air.rs:246-456), constraints in the reference's order."""
    local = bld.main().local
    # every initialisation input is boolean: inputs, chaining_values[0], [1], then counter_low, counter_hi, block_len, flags
    for c in range(INPUTS, INITIAL_ROW0):
        bld.assert_bool(local[c])
    # initial row0 = the packing of chaining_values[0]; initial row2 = IV[0..4]
    cv0 = [[local[chaining_values(0, j, i)] for i in range(32)] for j in range(4)]
    cv1 = [[local[chaining_values(1, j, i)] for i in range(32)] for j in range(4)]
    for j in range(4):
        bld.assert_eq(pack_bits_le(cv0[j][:16]), local[initial_row0(j, 0)])
        bld.assert_eq(pack_bits_le(cv0[j][16:]), local[initial_row0(j, 1)])
    for j in range(4):
        bld.assert_eq(local[initial_row2(j, 0)], IV[j] & 0xFFFF)
        bld.assert_eq(local[initial_row2(j, 1)], IV[j] >> 16)
    m = [[pack_bits_le([local[inputs(w, i)] for i in range(16)]), pack_bits_le([local[inputs(w, i)] for i in range(16, 32)])]
         for w in range(16)]
    row3_init = [[local[base + i] for i in range(32)] for base in (COUNTER_LOW, COUNTER_HI, BLOCK_LEN, FLAGS)]
    inp = _State([[local[initial_row0(j, l)] for l in range(2)] for j in range(4)], cv1,
                 [[local[initial_row2(j, l)] for l in range(2)] for j in range(4)], row3_init)
    for r in range(NUM_ROUNDS):
        rnd = [_trace_state(local, state(r, s)) for s in range(4)]
        _verify_round(bld, inp, rnd, m)
        m = [m[MSG_PERMUTATION[i]] for i in range(16)]                        # constants.rs permute, between rounds
        inp = rnd[STATE_OUTPUT]
    out = inp                                                                 # full_rounds[6].state_output
    helpers = [[local[final_round_helpers(j, i)] for i in range(32)] for j in range(4)]
    for j in range(4):
        bld.assert_eq(pack_bits_le(helpers[j][:16]), out.row2[j][0])
        bld.assert_eq(pack_bits_le(helpers[j][16:]), out.row2[j][1])
    o = [[[local[outputs(k, j, i)] for i in range(32)] for j in range(4)] for k in range(4)]
    for j in range(4):
        for i in range(32):
            bld.assert_bool(o[0][j][i])
    for j in range(4):
        xor_32_shift(bld, out.row0[j], o[0][j], helpers[j], 0)
    for k, left, right in ((1, out.row1, out.row3), (2, cv0, helpers), (3, cv1, out.row3)):
        for j in range(4):
            for i in range(32):
                bld.assert_eq(o[k][j][i], _xor(left[j][i], right[j][i]))


def random_inputs(n: int, seed: int = 1) -> np.ndarray:
    """(n, 24) uint32: `SmallRng::seed_from_u64(seed)` then `rng.random::<[u32; 24]>()` n times (blake3-air/src/air.rs:27-35).

    rand's SmallRng draws a u32 as the high half of one xoshiro256++ `next_u64`, so this is the u64 stream of
    keccak_air.random_inputs, shifted; the fixture replay pins this u32 draw."""
    from .keccak_air import random_inputs as u64_stream
    draws = u64_stream(-(-24 * n // 25), seed).ravel()[: 24 * n]
    return (draws >> np.uint64(32)).astype(np.uint32).reshape(n, 24)


class Blake3Air(KernelAir):
    """Blake3Air (blake3-air/src/air.rs) in the surface uni_stark.prove and verify read: width 9168, max_constraint_degree 3, no
    public values, main_next_row_columns() empty (the proof carries no next-row opening).  `gpu`: a plonky3_b200.gpu.Gpu (or None
    for a verifier-only AIR)."""
    air_name = "Blake3"

    def __init__(self, field: Field, gpu=None):
        super().__init__(field, WIDTH, eval_blake3, main_next_row_columns=[], max_constraint_degree=3, gpu=gpu)

    def generate_trace_rows(self, inputs_dev):
        """generate_trace_rows (blake3-air/src/generation.rs:16-118): (n, 24) device int32 tensor of u32 words (16 message words,
        then 8 chaining-value words), n a power of two -> the (n, 9168) device trace; row i hashes with counter i, block_len n,
        flags 0."""
        self._need_gpu("trace generation")
        return self.gpu.blake3_air_generate_trace(self.field.id, inputs_dev)

    def generate_random_trace_rows(self, n: int):
        """Blake3Air::generate_random_trace_rows(n, 0): the trace of `random_inputs(n)` (seed 1)."""
        import torch
        self._need_gpu("trace generation")
        x = self._to_device(torch.from_numpy(random_inputs(n).view(np.int32)))
        return self.generate_trace_rows(x)

    def generate_trace_cols(self, inputs_dev, col0: int, col1: int):
        """Columns [col0, col1) of `generate_trace_rows(inputs_dev)` without building the full trace: one rank's column block for
        `distributed.prove_sharded`."""
        self._need_gpu("trace generation")
        return self.gpu.blake3_air_generate_trace_cols(self.field.id, inputs_dev, int(col0), int(col1))

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        """`trace_lde_dev`: the trace on GENERATOR * K, |K| = 2N (the committed LDE's prefix).  Returns (2N, 4)."""
        return self.gpu.blake3_air_quotient(self.field.id, trace_lde_dev, int(log_degree), alpha)

    def _kernel_quotient_sharded(self, grp, log_lde_height: int, log_degree: int, alpha):
        return self.gpu.blake3_air_quotient_sharded(self.field.id, grp.struct, grp.col_starts, log_lde_height, log_degree, alpha)
