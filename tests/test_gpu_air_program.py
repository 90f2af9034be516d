"""Constraint programs on the GPU: `uni_stark.prove` of the DSL's Fibonacci AIR writes the reference's proof fixture byte for byte, the
quotient kernel (p3gpu_air_quotient_dev) equals the oracle (tests/air_oracle.py) on poisoned, guarded buffers over both fields, many
heights, quotient-domain sizes, widths and AIR shapes, the DSL's Poseidon2 AIR equals the hand-written kernel word for word and proves
the same bytes, MulAir proves and verifies at 2 and 4 quotient chunks, and errors are raised before anything launches."""
import json
import pathlib

import numpy as np
import pytest
import torch

import air_examples as E
import air_oracle as A
from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.air import SymbolicAir
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import Poseidon2, default_poseidon2
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air, poseidon2_eval
from plonky3_b200.uni_stark import StarkConfig, prove, verify
from plonky3_b200.verifier import VerificationError
from test_air_program_cpu import random_dag

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).resolve().parent / "golden"
GUARD = 64                                     # EF4 rows of 0xFFFFFFFF on each side of the output
POISON = np.uint32(0xFFFFFFFF)


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


def _p2_constants():
    oair = O.air_from_rng(KoalaBear.id, O.SmallRng(1))
    return oair, RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p], np.array(oair.end).reshape(4, 16))


# ---------------------------------------------------------------- the reference's Fibonacci proof
def test_fibonacci_proof_matches_the_reference_fixture(gpu):
    import fixture_replay as FR
    gold = json.loads((GOLD / "uni_stark_two_adic_v1.json").read_text())
    rc_i, rc_t, rc_p = FR.fixture_constants()
    pm = Poseidon2.new(BabyBear, 16, rc_i, rc_t, rc_p, monty=True)
    mmcs = MerkleTreeMmcs.poseidon2(pm, None, 0, gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(BabyBear, gpu), mmcs, FriParameters(2, 2, 1, 2, 1, 1, mmcs))     # fib_air.rs:134-155
    config = StarkConfig(pcs, pm, 8)                                                                         # DuplexChallenger<_, _, 16, 8>
    air = SymbolicAir(BabyBear, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    proof = prove(config, air, dev(E.fib_trace(BabyBear, 8)), [0, 1, 21])
    raw = proof.to_postcard()
    assert len(raw) == 1115 and raw.hex() == gold["postcard_hex"]
    verify(config, air, raw, [0, 1, 21])
    with pytest.raises(VerificationError):
        verify(config, air, raw, [0, 1, 22])


# ---------------------------------------------------------------- the kernel against the oracle
def _quotient_guarded(gpu, prog, lde_t, log_q, log_n, pubs, alpha):
    buf = torch.from_numpy(np.full(((1 << log_q) + 2 * GUARD, 4), POISON, dtype=np.uint32).view(np.int32)).cuda()
    out = buf[GUARD:GUARD + (1 << log_q)]
    gpu._use_torch_stream()
    pv = np.ascontiguousarray(pubs, dtype=np.uint32)
    H = int(lde_t.shape[0])
    _lib.check(gpu.L.p3gpu_air_quotient_dev(gpu.h, prog.h, lde_t.data_ptr(), H.bit_length() - 1, log_q, log_n,
                                            pv.ctypes.data if pv.size else None, np.ascontiguousarray(alpha, dtype=np.uint32).ctypes.data,
                                            out.data_ptr()))
    b = host(buf)
    assert (b[:GUARD] == POISON).all() and (b[GUARD + (1 << log_q):] == POISON).all(), "write outside the quotient"
    return b[GUARD:GUARD + (1 << log_q)]


def _compare(got, exp):
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"row {bad[0]}: got {got[bad[0]].tolist()} expected {exp[bad[0]].tolist()} ({bad.size} rows differ)"


def _check(gpu, f, nodes, cons, width, n_public, log_n, q, log_blowup, seed):
    rng = np.random.default_rng(seed)
    trace = f.to_monty_array(rng.integers(0, f.P, (1 << log_n, width)).astype(np.uint64)).astype(np.uint32)
    lde_t = gpu.coset_lde_batch(f.id, dev(trace), log_blowup, f.generator)
    pubs = [f.to_monty(int(v)) for v in rng.integers(0, f.P, n_public)]
    alpha = f.to_monty_array(rng.integers(0, f.P, 4).astype(np.uint64)).astype(np.uint32)
    prog = gpu.air_program_create(f.id, nodes, cons, width, n_public)
    got = _quotient_guarded(gpu, prog, lde_t, log_n + q, log_n, pubs, alpha)
    _compare(got, A.air_quotient(f.id, nodes, cons, host(lde_t), log_n + q, log_n, pubs, alpha))
    return prog


# (field, log_n, q, log_blowup, width, n_public, n_nodes, n_constraints)
RANDOM = [(BabyBear, 3, 1, 1, 3, 2, 60, 5), (KoalaBear, 3, 2, 3, 1, 0, 30, 3), (BabyBear, 4, 0, 1, 7, 1, 80, 9),
          (KoalaBear, 10, 1, 2, 33, 3, 400, 40), (BabyBear, 12, 2, 2, 64, 0, 600, 50), (KoalaBear, 16, 1, 1, 5, 1, 120, 10),
          (BabyBear, 20, 0, 1, 2, 2, 40, 4), (KoalaBear, 19, 1, 1, 3, 0, 50, 6), (BabyBear, 8, 3, 3, 2000, 2, 1500, 100)]


@pytest.mark.parametrize("case", RANDOM, ids=[f"{c[0].name}-n{c[1]}-q{c[2]}-w{c[4]}" for c in RANDOM])
def test_random_programs_match_oracle(gpu, case):
    f, log_n, q, lb, width, n_public, n_nodes, n_cons = case
    nodes, cons = random_dag(f, np.random.default_rng(log_n * 31 + width), width, n_public, n_nodes, n_cons)
    _check(gpu, f, nodes, cons, width, n_public, log_n, q, lb, seed=log_n)


def test_program_near_the_slot_limit(gpu):
    """380 values live at once: 380 products that every later constraint needs, summed first."""
    from plonky3_b200.air import ADD, MAIN_LOCAL, MAIN_NEXT, MUL
    f, width = KoalaBear, 380
    nodes = [(MAIN_LOCAL, c, 0, 0) for c in range(width)] + [(MAIN_NEXT, c, 0, 0) for c in range(width)]
    nodes += [(MUL, c, width + c, 0) for c in range(width)]
    acc = 2 * width
    for c in range(2 * width + 1, 3 * width):
        nodes.append((ADD, acc, c, 0)); acc = len(nodes) - 1
    cons = [acc] + list(range(2 * width, 3 * width))
    prog = _check(gpu, f, np.array(nodes), cons, width, 0, 6, 1, 1, seed=5)
    assert 380 <= prog.info()[1] <= 384


AIRS = ["fib", "mul3", "mul5_plain", "first_last_only", "transition_public"]


@pytest.mark.parametrize("name", AIRS)
@pytest.mark.parametrize("f", [BabyBear, KoalaBear])
def test_example_airs_match_oracle(gpu, f, name):
    def first_last(b):
        m = b.main()
        b.when_first_row().assert_zero(m.local[0] * m.local[1] - 7)
        b.when_last_row().assert_eq(m.local[1], m.local[0] + m.local[0])

    def trans_pub(b):
        m, p = b.main(), b.public_values()
        b.when_transition().assert_eq(m.next[0], m.local[0] * p[0] + p[1])
        b.assert_zero(-m.local[0] + p[1])
    air = {"fib": lambda: SymbolicAir(f, 2, E.fib_eval, 3),
           "mul3": lambda: SymbolicAir(f, 60, E.mul_air_eval(3, True, True)),
           "mul5_plain": lambda: SymbolicAir(f, 60, E.mul_air_eval(5, False, False)),
           "first_last_only": lambda: SymbolicAir(f, 2, first_last, main_next_row_columns=[]),
           "transition_public": lambda: SymbolicAir(f, 1, trans_pub, 2)}[name]()
    for log_n, q, lb in ((3, 0, 1), (5, 1, 2), (11, 2, 2), (14, 3, 3)):
        if q >= (max(air.max_constraint_degree(), 2) - 2).bit_length():
            _check(gpu, f, air.nodes, air.constraints, air.width(), air.num_public_values(), log_n, q, lb, seed=log_n + q)


# ---------------------------------------------------------------- against the hand-written Poseidon2 kernel
@pytest.mark.parametrize("log_n", [10, 12])
def test_poseidon2_program_equals_hand_written_kernel(gpu, log_n):
    oair, rc = _p2_constants()
    f = KoalaBear
    hand = VectorizedPoseidon2Air(f, rc, gpu)
    ev, width = poseidon2_eval(f, rc)
    dsl = SymbolicAir(f, width, ev, main_next_row_columns=[], gpu=gpu)
    inputs = O.random_matrix(f.id, 8 << log_n, 16, seed=log_n)
    trace = hand.generate_trace_rows(dev(inputs))
    lde = gpu.coset_lde_batch(f.id, trace, 1, f.generator)
    alpha = O.random_matrix(f.id, 1, 4, seed=9)[0]
    want = host(hand.quotient_values(lde, log_n, alpha))
    got = host(dsl.quotient_values(lde, log_n, alpha))
    _compare(got, want)


def _kb_config(gpu, log_blowup, num_queries=20, pow_bits=4):
    p16, p24 = default_poseidon2(KoalaBear, 16), default_poseidon2(KoalaBear, 24)
    mmcs = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=2, gpu=gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(KoalaBear, gpu), mmcs, FriParameters(log_blowup, 1, 3, num_queries, 0, pow_bits, mmcs))
    return StarkConfig(pcs, p24, 16)


def test_poseidon2_program_proves_the_same_bytes(gpu):
    oair, rc = _p2_constants()
    f, log_n = KoalaBear, 10
    p16, p24 = default_poseidon2(f, 16), default_poseidon2(f, 24)
    mmcs = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=3, gpu=gpu)
    config = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), mmcs, FriParameters(1, 0, 3, 30, 0, 8, mmcs)), p24, 16)
    hand = VectorizedPoseidon2Air(f, rc, gpu)
    ev, width = poseidon2_eval(f, rc)
    dsl = SymbolicAir(f, width, ev, main_next_row_columns=[], gpu=gpu)
    trace = hand.generate_trace_rows(dev(O.random_matrix(f.id, 8 << log_n, 16, seed=3)))
    raw = prove(config, hand, trace).to_postcard()
    assert prove(config, dsl, trace).to_postcard() == raw
    verify(config, dsl, raw)


# ---------------------------------------------------------------- round trips
@pytest.mark.parametrize("degree,log_blowup,chunks", [(3, 2, 2), (5, 3, 4)])
def test_mul_air_round_trip(gpu, degree, log_blowup, chunks):
    f, log_n = KoalaBear, 6
    config = _kb_config(gpu, log_blowup)
    air = SymbolicAir(f, 60, E.mul_air_eval(degree, True, True), gpu=gpu)
    trace = dev(E.mul_air_trace(f, 1 << log_n, degree, True, True))
    proof = prove(config, air, trace)
    assert len(proof.quotient_chunks) == chunks and proof.trace_next is not None
    raw = proof.to_postcard()
    verify(config, air, raw)
    for pos in (len(raw) // 5, len(raw) // 2, len(raw) - 30):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(config, air, bytes(bad))


# ---------------------------------------------------------------- errors: clean, before any launch
def test_errors_before_any_launch(gpu):
    f = KoalaBear
    trace = dev(E.mul_air_trace(f, 16, 5, False, False))
    config = _kb_config(gpu, 1)
    deg5 = SymbolicAir(f, 60, E.mul_air_eval(5, False, False), gpu=gpu)
    fib = SymbolicAir(f, 2, E.fib_eval, 3, gpu=gpu)
    fib_trace = dev(E.fib_trace(f, 16))
    lde = gpu.coset_lde_batch(f.id, fib_trace, 1, f.generator)
    n0 = gpu.launches
    with pytest.raises(ValueError, match="quotient chunks"):
        prove(config, deg5, trace)                                     # 4 chunks, blowup 2
    with pytest.raises(ValueError, match="public values"):
        prove(config, fib, fib_trace, [0, 1])
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.air_program_create(f.id, [(1, 0, 0, 0)], [0] * 2049, 1, 0)
    assert ex.value.code == _lib.EUNSUPPORTED and "2048" in str(ex.value)
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.air_program_create(f.id, [(1, 3, 0, 0)], [0], 2, 0)
    assert ex.value.code == _lib.EINVAL
    prog = gpu.air_program_create(f.id, fib.nodes, fib.constraints, 2, 3)
    with pytest.raises(_lib.P3GpuError) as ex:                         # quotient domain beyond the LDE
        gpu.air_quotient(prog, lde, 6, 4, [0, 1, 2], np.zeros(4, dtype=np.uint32))
    assert ex.value.code == _lib.EINVAL
    assert gpu.launches == n0
