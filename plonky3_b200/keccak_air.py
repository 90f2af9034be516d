"""The Keccak-f permutation AIR (keccak-air/src): the AIR of `prove_prime_field_31 --objective keccak-f-permutations`
(examples/src/airs.rs), over BabyBear and KoalaBear.

    air = KeccakAir(KoalaBear, gpu)
    trace = air.generate_random_trace_rows(43_690)           # or air.generate_trace_rows(inputs_dev), (n, 25) int64 on the device
    proof = uni_stark.prove(config, air, trace); uni_stark.verify(config, air, proof.to_postcard())

The constraints are written once, below, as a SymbolicAirBuilder eval that follows keccak-air/src/air.rs and round_flags.rs line
by line; the verifier folds them through SymbolicAir.eval_folded_constraints.  The prover does not use the constraint-program
kernel (3182 constraints are past its limit): trace generation and the quotient are the hand-written kernels of
csrc/keccak_air.cu (p3gpu_keccak_air_generate_trace_dev / p3gpu_keccak_air_quotient_dev), with no CPU fallback.

Column layout (columns.rs KeccakCols): step_flags [0,24) | export 24 | preimage [25,125) | a [125,225) | c [225,545) |
c_prime [545,865) | a_prime [865,2465) | a_prime_prime [2465,2565) | a_prime_prime_0_0_bits [2565,2629) |
a_prime_prime_prime_0_0_limbs [2629,2633).  preimage, a, a_prime and a_prime_prime are stored [y][x]; limbs are 16 bits, four
per u64, least significant first.
"""
from __future__ import annotations

import numpy as np

from .air import KernelAir
from .field import Field

NUM_ROUNDS, U64_LIMBS, BITS_PER_LIMB = 24, 4, 16
WIDTH = 2633
STEP_FLAGS, EXPORT, PREIMAGE, A, C, C_PRIME, A_PRIME = 0, 24, 25, 125, 225, 545, 865
A_PRIME_PRIME, A_PRIME_PRIME_0_0_BITS, A_PRIME_PRIME_PRIME_0_0_LIMBS = 2465, 2565, 2629
NEXT_ROW_READ = 225                    # the constraints read only step_flags, preimage and a of the next row: columns [0, 225)

R = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]   # constants.rs R[x][y]
RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
      0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
      0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
      0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]


# KeccakCols column indices (columns.rs)
def preimage(y, x, limb): return PREIMAGE + 4 * (5 * y + x) + limb
def a(y, x, limb): return A + 4 * (5 * y + x) + limb
def c(x, z): return C + 64 * x + z
def c_prime(x, z): return C_PRIME + 64 * x + z
def a_prime(y, x, z): return A_PRIME + 64 * (5 * y + x) + z
def a_prime_prime(y, x, limb): return A_PRIME_PRIME + 4 * (5 * y + x) + limb


def b(x, y, z):
    """columns.rs KeccakCols::b: B is a rotation of A', B[x, y] = ROT(A'[(x + 3y) % 5, x], R[(x + 3y) % 5][x])."""
    ax = (x + 3 * y) % 5
    return a_prime(x, ax, (z + 64 - R[ax][x]) % 64)


def a_prime_prime_prime(y, x, limb):
    return A_PRIME_PRIME_PRIME_0_0_LIMBS + limb if (y, x) == (0, 0) else a_prime_prime(y, x, limb)


def _xor(p, q): return p + q - p * (2 * q)           # PrimeCharacteristicRing::xor: x + y - x * 2y
def _xor3(p, q, r): return _xor(_xor(p, q), r)
def _andn(p, q): return (1 - p) * q


def _limb(bits):
    """(limb * 16 .. (limb + 1) * 16).rev().fold(0, |acc, z| acc.double() + bit(z)) over the limb's 16 bits, least significant first."""
    acc = None
    for v in reversed(bits):
        acc = v if acc is None else acc * 2 + v
    return acc


def eval_keccak(bld):
    """Air::eval for KeccakAir (keccak-air/src/air.rs:44-205), constraints in the reference's order."""
    main = bld.main()
    local, nxt = main.local, main.next
    # eval_round_flags (round_flags.rs:21-48)
    bld.when_first_row().assert_one(local[STEP_FLAGS])
    for i in range(1, NUM_ROUNDS):
        bld.when_first_row().assert_zero(local[STEP_FLAGS + i])
    for i in range(NUM_ROUNDS):
        bld.when_transition().assert_zero(local[STEP_FLAGS + i] - nxt[STEP_FLAGS + (i + 1) % NUM_ROUNDS])

    first_step = local[STEP_FLAGS]
    final_step = local[STEP_FLAGS + NUM_ROUNDS - 1]
    not_final_step = 1 - final_step
    transition_and_not_final = bld.is_transition() * not_final_step

    # If this is the first step, the input A must match the preimage.
    for y in range(5):
        for x in range(5):
            for limb in range(U64_LIMBS):
                bld.when(first_step).assert_zero(local[preimage(y, x, limb)] - local[a(y, x, limb)])
    # If this is not the final step, the local and next preimages must match.
    for y in range(5):
        for x in range(5):
            for limb in range(U64_LIMBS):
                bld.when(transition_and_not_final).assert_zero(local[preimage(y, x, limb)] - nxt[preimage(y, x, limb)])
    # The export flag must be 0 or 1, and 0 unless this is the final step.
    bld.assert_bool(local[EXPORT])
    bld.when(not_final_step).assert_zero(local[EXPORT])

    # C'[x, z] = xor(C[x, z], C[x - 1, z], C[x + 1, z - 1]).
    for x in range(5):
        for z in range(64):
            bld.assert_bool(local[c(x, z)])
        for z in range(64):
            xor = _xor3(local[c(x, z)], local[c((x + 4) % 5, z)], local[c((x + 1) % 5, (z + 63) % 64)])
            bld.assert_zero(local[c_prime(x, z)] - xor)

    # A[x, y, z] = xor(A'[x, y, z], C[x, z], C'[x, z]); every entry of A' is boolean.
    for x in range(5):
        c_xor_c_prime = [_xor(local[c(x, z)], local[c_prime(x, z)]) for z in range(64)]
        for y in range(5):
            for z in range(64):
                bld.assert_bool(local[a_prime(y, x, z)])
            for limb in range(U64_LIMBS):
                bits = [_xor(local[a_prime(y, x, z)], c_xor_c_prime[z]) for z in range(limb * BITS_PER_LIMB, (limb + 1) * BITS_PER_LIMB)]
                bld.assert_zero(_limb(bits) - local[a(y, x, limb)])

    # xor_{i=0}^4 A'[x, i, z] = C'[x, z]: diff (diff - 2) (diff - 4) = 0, diff = sum_i A'[x, i, z] - C'[x, z]
    for x in range(5):
        four = bld.constant(2) * 2
        for z in range(64):
            s = local[a_prime(0, x, z)]
            for y in range(1, 5):
                s = s + local[a_prime(y, x, z)]
            diff = s - local[c_prime(x, z)]
            bld.assert_zero(diff * (diff - 2) * (diff - four))

    # A''[x, y] = xor(B[x, y], andn(B[x + 1, y], B[x + 2, y])).
    for y in range(5):
        for x in range(5):
            def get_bit(z):
                andn = _andn(local[b((x + 1) % 5, y, z)], local[b((x + 2) % 5, y, z)])
                return _xor(andn, local[b(x, y, z)])
            for limb in range(U64_LIMBS):
                bits = [get_bit(z) for z in range(limb * BITS_PER_LIMB, (limb + 1) * BITS_PER_LIMB)]
                bld.assert_zero(_limb(bits) - local[a_prime_prime(y, x, limb)])

    # A'''[0, 0] = A''[0, 0] XOR RC; the bits of A''[0, 0] are boolean.
    for z in range(64):
        bld.assert_bool(local[A_PRIME_PRIME_0_0_BITS + z])
    for limb in range(U64_LIMBS):
        bits = [local[A_PRIME_PRIME_0_0_BITS + z] for z in range(limb * BITS_PER_LIMB, (limb + 1) * BITS_PER_LIMB)]
        bld.assert_zero(_limb(bits) - local[a_prime_prime(0, 0, limb)])

    def get_xored_bit(i):
        rc_bit_i = None
        for r in range(NUM_ROUNDS):
            if (RC[r] >> i) & 1:
                rc_bit_i = local[STEP_FLAGS + r] if rc_bit_i is None else rc_bit_i + local[STEP_FLAGS + r]
        if rc_bit_i is None:
            rc_bit_i = bld.constant(0)
        return _xor(rc_bit_i, local[A_PRIME_PRIME_0_0_BITS + i])

    for limb in range(U64_LIMBS):
        bits = [get_xored_bit(z) for z in range(limb * BITS_PER_LIMB, (limb + 1) * BITS_PER_LIMB)]
        bld.assert_zero(_limb(bits) - local[A_PRIME_PRIME_PRIME_0_0_LIMBS + limb])

    # Enforce that this round's output equals the next round's input (x-outer, y-inner).
    for x in range(5):
        for y in range(5):
            for limb in range(U64_LIMBS):
                bld.when(transition_and_not_final).assert_zero(local[a_prime_prime_prime(y, x, limb)] - nxt[a(y, x, limb)])


def random_inputs(n: int, seed: int = 1) -> np.ndarray:
    """(n, 25) uint64: `SmallRng::seed_from_u64(seed)` then `rng.random::<[u64; 25]>()` n times (keccak-air/src/air.rs:25-33).

    Restates rand 0.10's SmallRng on 64-bit targets, xoshiro256++ (`Xoshiro256PlusPlus::seed_from_u64`: four SplitMix64 outputs;
    `next_u64`), and the StandardUniform draws of a u64 (one `next_u64`) and of an array (its elements in order).  The seeding and
    the u32 draw are the ones the fixture replay pins; no published known answer exists for the u64 draw, so this sequence is
    unverified against the reference."""
    M = (1 << 64) - 1
    s, x = [], seed & M
    for _ in range(4):
        x = (x + 0x9E3779B97F4A7C15) & M
        z = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        s.append(z ^ (z >> 31))
    s0, s1, s2, s3 = s
    out = np.empty(25 * n, dtype=np.uint64)
    for k in range(25 * n):
        t = (s0 + s3) & M
        out[k] = (((t << 23) | (t >> 41)) + s0) & M
        t = (s1 << 17) & M
        s2 ^= s0; s3 ^= s1; s1 ^= s2; s0 ^= s3; s2 ^= t
        s3 = ((s3 << 45) | (s3 >> 19)) & M
    return out.reshape(n, 25)


class KeccakAir(KernelAir):
    """KeccakAir (keccak-air/src/air.rs) in the surface uni_stark.prove and verify read: width 2633, max_constraint_degree 3 (the
    DAG's), no public values, every column opened at the next point (BaseAir's default main_next_row_columns, which KeccakAir
    keeps).  `gpu`: a plonky3_b200.gpu.Gpu (or None for a verifier-only AIR)."""
    air_name = "Keccak"

    def __init__(self, field: Field, gpu=None):
        super().__init__(field, WIDTH, eval_keccak, gpu=gpu)

    def generate_trace_rows(self, inputs_dev):
        """generate_trace_rows (keccak-air/src/generation.rs:16-64): (n, 25) device int64 tensor of u64 lanes, input[x + 5 y] =
        state[x][y] -> the ((24 n).next_power_of_two(), 2633) device trace, padding included."""
        self._need_gpu("trace generation")
        return self.gpu.keccak_air_generate_trace(self.field.id, inputs_dev)

    def generate_random_trace_rows(self, n: int):
        """KeccakAir::generate_random_trace_rows(n, 0): the trace of `random_inputs(n)` (seed 1)."""
        import torch
        self._need_gpu("trace generation")
        x = self._to_device(torch.from_numpy(random_inputs(n).view(np.int64)))
        return self.generate_trace_rows(x)

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        """`trace_lde_dev`: the trace on GENERATOR * K, |K| = 2N (the committed LDE's prefix).  Returns (2N, 4)."""
        return self.gpu.keccak_air_quotient(self.field.id, trace_lde_dev, int(log_degree), alpha)
