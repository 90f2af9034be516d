"""The SHA-256 compression AIR (sha256-air/src), over BabyBear and KoalaBear.

    air = Sha256Air(KoalaBear, gpu)
    trace = air.generate_random_trace_rows(1 << 18)           # or air.generate_trace_rows(inputs_dev), (n, 24) int32 on the device
    proof = uni_stark.prove(config, air, trace); uni_stark.verify(config, air, proof.to_postcard())

One row per compression, rows independent: no selectors, no next-row reads, no public values.  The constraints are written once,
below, as a SymbolicAirBuilder eval that follows sha256-air/src/air.rs line by line; the verifier folds them through
SymbolicAir.eval_folded_constraints.  The prover does not use the constraint-program kernel (8096 constraints are past its limit):
trace generation and the quotient are the hand-written kernels of csrc/sha256_air.cu (p3gpu_sha256_air_generate_trace_dev /
p3gpu_sha256_air_quotient_dev), with no CPU fallback.

Column layout (columns.rs Sha256Cols, repr(C)): h_in [8][2] limbs [0,16) | a_chain [68][32] bits [16,2192) | e_chain [68][32]
[2192,4368) | w [64][32] [4368,6416) | sched_sigma0, sched_sigma1, sched_tmp [48][2] each [6416,6704) | rounds [64] x (sigma1_e, ch,
tmp1, t1, sigma0_a, maj) [2] each [6704,7472) | h_out [8][32] bits [7472,7728).  Bits are least significant first, limbs [lo, hi].
a_chain[0..4] holds H3, H2, H1, H0 and a_chain[t + 4] round t's new a (e_chain likewise with H7..H4 and new e), so round t reads
a, b, c, d = a_chain[t + 3], [t + 2], [t + 1], [t] and e, f, g, h from e_chain.
"""
from __future__ import annotations

import numpy as np

from .air import KernelAir
from .blake3_air import _xor, add2, add3, pack_bits_le
from .field import Field

WIDTH = 7728
NUM_ROUNDS, BLOCK_WORDS, STATE_WORDS, CHAIN_LEN = 64, 16, 8, 68
SCHEDULE_EXTENSIONS = NUM_ROUNDS - BLOCK_WORDS
H_IN, A_CHAIN, E_CHAIN, W = 0, 16, 2192, 4368
SCHED_SIGMA0, SCHED_SIGMA1, SCHED_TMP, ROUNDS, H_OUT = 6416, 6512, 6608, 6704, 7472
ROUND_WIDTH = 12
SIGMA1_E, CH, TMP1, T1, SIGMA0_A, MAJ = 0, 2, 4, 6, 8, 10     # a round's packed fields, in column order

K = [0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,   # constants.rs SHA256_K
     0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
     0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
     0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
     0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
     0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
     0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
     0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2]
IV = [0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19]

# sigma_params (air.rs): (r1, r2, r3, third operand is a logical shift)
BIG_SIGMA0, BIG_SIGMA1, SMALL_SIGMA0, SMALL_SIGMA1 = (2, 13, 22, False), (6, 11, 25, False), (7, 18, 3, True), (17, 19, 10, True)


# Sha256Cols column indices (columns.rs)
def h_in(i, limb): return H_IN + 2 * i + limb
def a_chain(j, b): return A_CHAIN + 32 * j + b
def e_chain(j, b): return E_CHAIN + 32 * j + b
def w(t, b): return W + 32 * t + b
def sched_sigma0(i, limb): return SCHED_SIGMA0 + 2 * i + limb
def sched_sigma1(i, limb): return SCHED_SIGMA1 + 2 * i + limb
def sched_tmp(i, limb): return SCHED_TMP + 2 * i + limb
def rounds(t, field, limb): return ROUNDS + ROUND_WIDTH * t + field + limb
def h_out(i, b): return H_OUT + 32 * i + b


def _pack_word(bits):
    """air.rs pack_word: [lo, hi] of 32 bits."""
    return [pack_bits_le(bits[:16]), pack_bits_le(bits[16:])]


def _assert_packed(bld, packed, built):
    """packed - built, one constraint per limb (assert_packed_equals_bits and the tails of the sigma / Ch / Maj checks)."""
    bld.assert_zero(packed[0] - built[0])
    bld.assert_zero(packed[1] - built[1])


def _sigma(bld, bits, spec, packed):
    """air.rs assert_sigma_matches: bit i of the output is bits[i + r1] ^ bits[i + r2] ^ bits[i + r3] (indices mod 32; for a
    logical shift a third index past 31 reads zero, and xor with zero is the identity)."""
    r1, r2, r3, shr = spec
    out = []
    for i in range(32):
        v = _xor(bits[(i + r1) % 32], bits[(i + r2) % 32])
        if not (shr and i + r3 >= 32):
            v = _xor(v, bits[(i + r3) % 32])
        out.append(v)
    _assert_packed(bld, packed, _pack_word(out))


def eval_sha256(bld):
    """Air::eval for Sha256Air (sha256-air/src/air.rs), constraints in the reference's order."""
    local = bld.main().local
    wb = [[local[w(t, b)] for b in range(32)] for t in range(NUM_ROUNDS)]
    ab = [[local[a_chain(j, b)] for b in range(32)] for j in range(CHAIN_LEN)]
    eb = [[local[e_chain(j, b)] for b in range(32)] for j in range(CHAIN_LEN)]
    ob = [[local[h_out(i, b)] for b in range(32)] for i in range(STATE_WORDS)]
    hin = [[local[h_in(i, l)] for l in range(2)] for i in range(STATE_WORDS)]
    # eval_bit_range_checks: w, a_chain, e_chain, h_out
    for words in (wb, ab, eb, ob):
        for word in words:
            for v in word:
                bld.assert_bool(v)
    # eval_initial_state: H_i against a_chain[3 - i], H_{4+i} against e_chain[3 - i]
    for chain, off in ((ab, 0), (eb, 4)):
        for i in range(4):
            _assert_packed(bld, hin[off + i], _pack_word(chain[3 - i]))
    # eval_message_schedule
    for i in range(SCHEDULE_EXTENSIONS):
        t = i + BLOCK_WORDS
        s0 = [local[sched_sigma0(i, l)] for l in range(2)]
        s1 = [local[sched_sigma1(i, l)] for l in range(2)]
        tmp = [local[sched_tmp(i, l)] for l in range(2)]
        _sigma(bld, wb[t - 15], SMALL_SIGMA0, s0)
        _sigma(bld, wb[t - 2], SMALL_SIGMA1, s1)
        add2(bld, tmp, s1, _pack_word(wb[t - 7]))
        add3(bld, _pack_word(wb[t]), tmp, s0, _pack_word(wb[t - 16]))        # add3_expr_out
    # eval_compression
    for t in range(NUM_ROUNDS):
        a, b, c, d = ab[t + 3], ab[t + 2], ab[t + 1], ab[t]
        e, f, g, h = eb[t + 3], eb[t + 2], eb[t + 1], eb[t]
        col = lambda fld: [local[rounds(t, fld, l)] for l in range(2)]
        sigma1_e, ch, tmp1, t1, sigma0_a, maj = (col(x) for x in (SIGMA1_E, CH, TMP1, T1, SIGMA0_A, MAJ))
        _sigma(bld, e, BIG_SIGMA1, sigma1_e)
        _assert_packed(bld, ch, _pack_word([e[i] * f[i] + (1 - e[i]) * g[i] for i in range(32)]))     # assert_ch_matches
        add3(bld, tmp1, sigma1_e, ch, _pack_word(h))
        add3(bld, t1, tmp1, [K[t] & 0xFFFF, K[t] >> 16], _pack_word(wb[t]))
        _sigma(bld, a, BIG_SIGMA0, sigma0_a)
        _assert_packed(bld, maj, _pack_word([a[i] * b[i] + c[i] * _xor(a[i], b[i]) for i in range(32)]))   # assert_maj_matches
        add3(bld, _pack_word(ab[t + 4]), t1, sigma0_a, maj)                      # add3_expr_out
        add2(bld, _pack_word(eb[t + 4]), t1, _pack_word(d))                      # add2_expr_out
    # eval_finalization: H'_i = H_i + a_chain[67 - i], H'_{4+i} = H_{4+i} + e_chain[67 - i]
    for chain, off in ((ab, 0), (eb, 4)):
        for i in range(4):
            add2(bld, _pack_word(ob[off + i]), hin[off + i], _pack_word(chain[CHAIN_LEN - 1 - i]))


def random_inputs(n: int, seed: int = 1) -> np.ndarray:
    """(n, 24) uint32: `SmallRng::seed_from_u64(seed)` then `rng.random::<[u32; 24]>()` n times (Sha256Air::generate_trace_rows),
    the draw of blake3_air.random_inputs."""
    from .blake3_air import random_inputs as u32_draw
    return u32_draw(n, seed)


class Sha256Air(KernelAir):
    """Sha256Air (sha256-air/src/air.rs) in the surface uni_stark.prove and verify read: width 7728, max_constraint_degree 3, no
    public values, main_next_row_columns() empty (the proof carries no next-row opening).  `gpu`: a plonky3_b200.gpu.Gpu (or None
    for a verifier-only AIR)."""
    air_name = "SHA-256"

    def __init__(self, field: Field, gpu=None):
        super().__init__(field, WIDTH, eval_sha256, main_next_row_columns=[], max_constraint_degree=3, gpu=gpu)

    def generate_trace_rows(self, inputs_dev):
        """generate_trace_rows (sha256-air/src/generation.rs): (n, 24) device int32 tensor of u32 words (the 16-word block, then the
        8-word chaining state), n a power of two -> the (n, 7728) device trace."""
        self._need_gpu("trace generation")
        return self.gpu.sha256_air_generate_trace(self.field.id, inputs_dev)

    def generate_random_trace_rows(self, n: int):
        """Sha256Air::generate_trace_rows(n, _): the trace of `random_inputs(n)` (seed 1)."""
        import torch
        self._need_gpu("trace generation")
        x = self._to_device(torch.from_numpy(random_inputs(n).view(np.int32)))
        return self.generate_trace_rows(x)

    def generate_trace_cols(self, inputs_dev, col0: int, col1: int):
        """Columns [col0, col1) of `generate_trace_rows(inputs_dev)` without building the full trace: one rank's column block for
        `distributed.prove_sharded`."""
        self._need_gpu("trace generation")
        return self.gpu.sha256_air_generate_trace_cols(self.field.id, inputs_dev, int(col0), int(col1))

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        """`trace_lde_dev`: the trace on GENERATOR * K, |K| = 2N (the committed LDE's prefix).  Returns (2N, 4)."""
        return self.gpu.sha256_air_quotient(self.field.id, trace_lde_dev, int(log_degree), alpha)

    def _kernel_quotient_sharded(self, grp, log_lde_height: int, log_degree: int, alpha):
        return self.gpu.sha256_air_quotient_sharded(self.field.id, grp.struct, grp.col_starts, log_lde_height, log_degree, alpha)
