"""Constraint programs on the CPU: the DSL's degree inference (plonky3_b200.air) against the reference's values, the compiler and the
per-instruction semantics of csrc/air_program.cuh (run on the host by tests/cpp/air_program_check.cpp) against the independent oracle
(tests/air_oracle.py), node-list validation, the verifier's folder on the same DAG, and the product `prove` driver writing the reference's
Fibonacci proof fixture byte for byte with every device call answered on the CPU."""
import copy
import json
import os
import pathlib
import subprocess

import numpy as np
import pytest
import torch

import air_examples as E
import air_oracle as A
from plonky3_b200 import _lib
from plonky3_b200.air import (ADD, CONST, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, MAIN_LOCAL, MAIN_NEXT, MUL, NEG, PUBLIC, SUB,
                              SymbolicAir)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air, poseidon2_eval
from plonky3_b200.uni_stark import get_log_num_quotient_chunks

ROOT = pathlib.Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = tmp_path_factory.mktemp("air") / "air_program_check"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "air_program_check.cpp"), "-o", str(exe)],
                   check=True)
    return exe


def _job(mode, field, width, n_public, nodes, cons):
    nodes = np.asarray(nodes, dtype=np.uint32).reshape(-1, 4)
    cons = np.asarray(cons, dtype=np.uint32).ravel()
    return [mode, field.id, width, n_public, nodes.shape[0], cons.size, *nodes.ravel().tolist(), *cons.tolist()]


def run_compile(exe, field, width, n_public, nodes, cons):
    out = subprocess.run([str(exe)], input=" ".join(map(str, _job("c", field, width, n_public, nodes, cons))), capture_output=True, text=True,
                         check=True).stdout.split()
    return tuple(int(v) for v in out[:4])            # rc, instructions, slots, max_live


def run_quotient(exe, field, width, n_public, nodes, cons, lde, log_q, log_n, pubs, alpha):
    job = _job("q", field, width, n_public, nodes, cons) + [log_q, log_n, *np.asarray(lde)[: 1 << log_q].ravel().tolist(),
                                                             *list(pubs), *np.asarray(alpha).tolist()]
    out = subprocess.run([str(exe)], input=" ".join(map(str, job)), capture_output=True, text=True, check=True).stdout.split("\n")
    head = tuple(int(v) for v in out[0].split())
    return head, np.array(out[1].split(), dtype=np.uint32).reshape(-1, 4)


def random_dag(field, rng, width, n_public, n_nodes, n_cons, chain=False):
    """A random node list: leaves of every kind, then operations on random earlier nodes (or a deep chain)."""
    nodes = []
    for k in range(min(8, n_nodes)):
        kind = k % 8
        if kind in (0, 1):
            nodes.append((MAIN_LOCAL, int(rng.integers(width)), 0, 0))
        elif kind == 2:
            nodes.append((MAIN_NEXT, int(rng.integers(width)), 0, 0))
        elif kind == 3:
            nodes.append((CONST, 0, 0, field.to_monty(int(rng.integers(field.P)))))
        elif kind == 4 and n_public:
            nodes.append((PUBLIC, int(rng.integers(n_public)), 0, 0))
        elif kind == 5:
            nodes.append((IS_FIRST_ROW, 0, 0, 0))
        elif kind == 6:
            nodes.append((IS_LAST_ROW, 0, 0, 0))
        else:
            nodes.append((IS_TRANSITION, 0, 0, 0))
    while len(nodes) < n_nodes:
        i = len(nodes)
        op = int(rng.choice([ADD, SUB, MUL, NEG, MAIN_LOCAL]))
        if op == MAIN_LOCAL:
            nodes.append((MAIN_LOCAL, int(rng.integers(width)), 0, 0))
        elif chain:
            nodes.append((op, i - 1, int(rng.integers(i)), 0))
        else:
            nodes.append((op, int(rng.integers(i)), int(rng.integers(i)), 0))
    cons = [int(v) for v in rng.integers(0, n_nodes, n_cons)]
    return np.array(nodes, dtype=np.uint32), cons


def _inputs(field, rng, width, n_public, log_q):
    lde = field.to_monty_array(rng.integers(0, field.P, (1 << log_q, width)).astype(np.uint64)).astype(np.uint32)
    pubs = [field.to_monty(int(v)) for v in rng.integers(0, field.P, n_public)]
    alpha = field.to_monty_array(rng.integers(0, field.P, 4).astype(np.uint64)).astype(np.uint32)
    return lde, pubs, alpha


def _p2_constants():
    from oracle import p3_oracle as O
    oair = O.air_from_rng(KoalaBear.id, O.SmallRng(1))
    return RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p], np.array(oair.end).reshape(4, 16))


# ---------------------------------------------------------------- degrees
def test_degree_inference_matches_the_reference():
    fib = SymbolicAir(BabyBear, 2, E.fib_eval, num_public_values=3)
    assert (fib.max_constraint_degree(), get_log_num_quotient_chunks(fib)) == (2, 0)
    assert fib.main_next_row_columns() == [0, 1]                      # BaseAir default: every column
    for d in range(2, 7):
        for boundary in (False, True):
            for transition in (False, True):
                air = SymbolicAir(BabyBear, 60, E.mul_air_eval(d, boundary, transition))
                deg = max(d, 3) if boundary else d                   # first_row (deg 1) * (a * a + 1 - b)
                assert air.max_constraint_degree() == deg
                assert get_log_num_quotient_chunks(air) == (deg - 1 - 1).bit_length()     # log2_ceil(deg - 1)
                assert len(air.constraints) == 20 * (1 + boundary + transition)
    ev, width = poseidon2_eval(KoalaBear, _p2_constants())
    p2 = SymbolicAir(KoalaBear, width, ev, main_next_row_columns=[])
    assert (width, p2.max_constraint_degree(), len(p2.constraints), get_log_num_quotient_chunks(p2)) == (1312, 3, 8 * 148, 1)
    # a hint overrides the inferred degree (uni-stark/src/symbolic.rs)
    assert get_log_num_quotient_chunks(SymbolicAir(BabyBear, 2, E.fib_eval, 3, max_constraint_degree=5)) == 2


def test_builder_shares_identical_subexpressions():
    def ev(b):
        m = b.main()
        x = (m.local[0] + 3) * m.local[1]
        y = (m.local[0] + 3) * m.local[1]
        assert x.i == y.i
        b.assert_zero(x - y)
        b.when(m.local[0]).when_transition().assert_one(m.next[0])
    air = SymbolicAir(KoalaBear, 2, ev)
    assert len(air.nodes) == len({tuple(n) for n in air.nodes.tolist()})
    assert air.constraint_degrees() == [2, 2]


# ---------------------------------------------------------------- compiler + instruction semantics on the host vs the oracle
CASES = [(f, seed, shape) for f in (BabyBear, KoalaBear) for seed, shape in
         [(1, (5, 1, 40, 6, 3, 2)), (2, (9, 2, 200, 25, 4, 1)), (3, (3, 0, 120, 1, 2, 0)), (4, (17, 3, 400, 60, 5, 3))]]


@pytest.mark.parametrize("f,seed,shape", CASES, ids=[f"{c[0].name}-{c[1]}" for c in CASES])
def test_random_dags_match_oracle(checker, f, seed, shape):
    width, n_public, n_nodes, n_cons, log_n, q = shape
    rng = np.random.default_rng(seed)
    nodes, cons = random_dag(f, rng, width, n_public, n_nodes, n_cons)
    lde, pubs, alpha = _inputs(f, rng, width, n_public, log_n + q)
    (rc, n_insn, slots, live), got = run_quotient(checker, f, width, n_public, nodes, cons, lde, log_n + q, log_n, pubs, alpha)
    assert rc == 0
    exp = A.air_quotient(f.id, nodes, cons, lde, log_n + q, log_n, pubs, alpha)
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"first differing row {bad[:1]}"
    # the oracle in chunks of 3 natural indices (each gathering its own rows, next rows and selectors) gives the same words
    assert np.array_equal(A.air_quotient(f.id, nodes, cons, lde, log_n + q, log_n, pubs, alpha, chunk_points=3), exp)
    reachable = n_insn - len(cons)                                    # every emitted compute instruction is one live node
    assert slots == live <= reachable


@pytest.mark.parametrize("f", [BabyBear, KoalaBear])
def test_deep_chains_reuse_slots(checker, f):
    rng = np.random.default_rng(7)
    nodes, cons = random_dag(f, rng, 4, 1, 3000, 2, chain=True)
    cons = [2999, 1500]
    lde, pubs, alpha = _inputs(f, rng, 4, 1, 4)
    (rc, n_insn, slots, live), got = run_quotient(checker, f, 4, 1, nodes, cons, lde, 4, 3, pubs, alpha)
    assert rc == 0 and slots == live
    assert slots < 200 < n_insn                                       # far fewer slots than values
    assert np.array_equal(got, A.air_quotient(f.id, nodes, cons, lde, 4, 3, pubs, alpha))
    # a pure chain: at most 3 values live at once
    chain = [(MAIN_LOCAL, 0, 0, 0)] + [(MUL if k % 2 else ADD, k - 1, k - 1, 0) for k in range(1, 5000)]
    rc, n_insn, slots, live = run_compile(checker, f, 1, 0, chain, [4999])
    assert (rc, n_insn, slots) == (0, 5001, 1)


def _example_airs():
    p2_ev, p2_w = poseidon2_eval(KoalaBear, _p2_constants(), vector_len=1)
    return {
        "fibonacci": (BabyBear, SymbolicAir(BabyBear, 2, E.fib_eval, 3), 3, 0),
        "mul_air_3": (BabyBear, SymbolicAir(BabyBear, 60, E.mul_air_eval(3, True, True)), 4, 1),
        "mul_air_5_plain": (KoalaBear, SymbolicAir(KoalaBear, 60, E.mul_air_eval(5, False, False)), 4, 2),
        "mul_air_6": (KoalaBear, SymbolicAir(KoalaBear, 60, E.mul_air_eval(6, True, True)), 3, 3),
        "poseidon2_vec1": (KoalaBear, SymbolicAir(KoalaBear, p2_w, p2_ev, main_next_row_columns=[]), 3, 1),
    }


@pytest.mark.parametrize("name", ["fibonacci", "mul_air_3", "mul_air_5_plain", "mul_air_6", "poseidon2_vec1"])
def test_example_airs_match_oracle(checker, name):
    f, air, log_n, q = _example_airs()[name]
    rng = np.random.default_rng(11)
    lde, pubs, alpha = _inputs(f, rng, air.width(), air.num_public_values(), log_n + q)
    (rc, n_insn, slots, live), got = run_quotient(checker, f, air.width(), air.num_public_values(), air.nodes, air.constraints, lde,
                                                  log_n + q, log_n, pubs, alpha)
    assert rc == 0 and slots == live
    exp = A.air_quotient(f.id, air.nodes, air.constraints, lde, log_n + q, log_n, pubs, alpha)
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"first differing row {bad[:1]}"


def test_oracle_quotient_is_low_degree_on_a_valid_trace():
    """Sanity of the oracle: on a valid Fibonacci trace the quotient has degree < (d - 1) N."""
    from oracle import p3_oracle as O
    air = SymbolicAir(BabyBear, 2, E.fib_eval, 3)
    trace = E.fib_trace(BabyBear, 16)
    lde = O.coset_lde_batch(0, trace, 2, BabyBear.generator, bitrev_out=True)
    pubs = [BabyBear.to_monty(v) for v in (0, 1, BabyBear.from_monty(int(trace[-1, 1])))]
    alpha = BabyBear.to_monty_array(np.array([3, 5, 7, 11], dtype=np.uint64)).astype(np.uint32)
    q = A.air_quotient(0, air.nodes, air.constraints, lde, 4, 4, pubs, alpha)
    assert not O.coset_idft_batch(0, q, BabyBear.generator)[15:].any()
    pubs[2] = BabyBear.to_monty(5)
    q = A.air_quotient(0, air.nodes, air.constraints, lde, 4, 4, pubs, alpha)
    assert O.coset_idft_batch(0, q, BabyBear.generator)[15:].any()


# ---------------------------------------------------------------- validation
def test_bad_node_lists_are_rejected(checker):
    f = KoalaBear
    ok = [(MAIN_LOCAL, 0, 0, 0), (PUBLIC, 0, 0, 0), (SUB, 0, 1, 0)]
    assert run_compile(checker, f, 2, 1, ok, [2])[0] == 0
    bad = [
        ([(MAIN_LOCAL, 2, 0, 0)], [0], _lib.EINVAL),                          # column >= width
        ([(MAIN_NEXT, 5, 0, 0)], [0], _lib.EINVAL),
        ([(PUBLIC, 1, 0, 0)], [0], _lib.EINVAL),                              # public index >= n_public
        ([(MAIN_LOCAL, 0, 0, 0), (ADD, 0, 1, 0)], [1], _lib.EINVAL),         # forward (self) operand
        ([(MAIN_LOCAL, 0, 0, 0), (NEG, 7, 0, 0)], [1], _lib.EINVAL),         # out-of-range operand
        ([(MAIN_LOCAL, 0, 0, 0), (12, 0, 0, 0)], [1], _lib.EINVAL),          # unknown op
        ([(CONST, 0, 0, f.P)], [0], _lib.EINVAL),                            # constant not canonical
        (ok, [3], _lib.EINVAL),                                              # constraint names no node
    ]
    for nodes, cons, code in bad:
        assert run_compile(checker, f, 2, 1, nodes, cons)[0] == code, nodes
    assert run_compile(checker, BabyBear, 2, 1, ok, [2])[0] == 0
    job = _job("c", f, 2, 1, ok, [2]); job[1] = 7                            # unsupported field
    out = subprocess.run([str(checker)], input=" ".join(map(str, job)), capture_output=True, text=True, check=True).stdout.split()
    assert int(out[0]) == _lib.EUNSUPPORTED


def test_limits_are_unsupported(checker):
    f = BabyBear
    # 2049 constraints
    assert run_compile(checker, f, 1, 0, [(MAIN_LOCAL, 0, 0, 0)], [0] * 2049)[0] == _lib.EUNSUPPORTED
    assert run_compile(checker, f, 1, 0, [(MAIN_LOCAL, 0, 0, 0)], [0] * 2048)[0] == 0
    # 400 values that all stay live for later constraints: more than 384 slots
    nodes = [(MAIN_LOCAL, c, 0, 0) for c in range(400)]
    nodes += [(MUL, c, c, 0) for c in range(400)]
    acc = 400
    for c in range(401, 800):
        nodes.append((ADD, acc, c, 0)); acc = len(nodes) - 1
    cons = [acc] + list(range(400, 800))
    assert run_compile(checker, f, 400, 0, nodes, cons)[0] == _lib.EUNSUPPORTED
    rc, _, slots, _ = run_compile(checker, f, 400, 0, nodes[:700] + [(ADD, 400, 401, 0)], [700] + list(range(400, 700)))
    assert rc == 0 and slots <= 384


# ---------------------------------------------------------------- the verifier's folder on the same DAG
def test_folder_matches_hand_written_fibonacci():
    import stark_verify as V
    from plonky3_b200.verifier import Ext
    e = Ext(BabyBear)
    air = SymbolicAir(BabyBear, 2, E.fib_eval, 3)
    rng = np.random.default_rng(3)
    ef = lambda: [int(v) for v in rng.integers(0, BabyBear.P, 4)]
    for _ in range(20):
        args = ([ef(), ef()], [ef(), ef()], [int(v) for v in rng.integers(0, BabyBear.P, 3)], ef(), ef(), ef(), ef())
        assert air.eval_folded_constraints(e, *args) == V.FibonacciAir().eval_folded_constraints(e, *args)
    # the Poseidon2 AIR's folder (its builder eval through SymbolicAir) against the restated verifier's, on random opened rows
    from oracle import p3_oracle as O
    oair = O.air_from_rng(KoalaBear.id, O.SmallRng(1))
    p2 = VectorizedPoseidon2Air(KoalaBear, RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p],
                                                          np.array(oair.end).reshape(4, 16)), None)
    fold, fld = V.poseidon2_air(oair)["constraints"], V.Fld(KoalaBear.id)
    ef = lambda: [int(v) for v in rng.integers(0, KoalaBear.P, 4)]
    for _ in range(3):
        args = ([ef() for _ in range(p2.width())], [], [], ef(), ef(), ef(), ef())
        assert p2.eval_folded_constraints(Ext(KoalaBear), *args) == fold(fld, *args)


def test_next_row_needs_next_columns():
    with pytest.raises(ValueError, match="next row"):
        SymbolicAir(BabyBear, 2, E.fib_eval, 3, main_next_row_columns=[])


# ---------------------------------------------------------------- the prove driver writes the reference's fixture
class BabyBearChallenger:
    """DuplexChallenger<BabyBear, Poseidon2-16, 16, 8> on the oracle permutation, in the product challenger's surface."""

    def __init__(self, perm):
        import stark_verify as V
        self.f = V.Fld(BabyBear.id)
        self.ch = V.Challenger(self.f, perm, 16, 8)

    def observe(self, word): self.ch.observe(self.f.c(word))
    def observe_canonical(self, x): self.ch.observe(int(x))
    def observe_slice(self, words): self.ch.observe_words(np.asarray(words.numpy() if hasattr(words, "numpy") else words).view(np.uint32)
                                                          if hasattr(words, "numpy") else words)
    def observe_cap(self, cap): self.observe_slice(cap)
    def observe_algebra_slice(self, ys): self.observe_slice(ys)
    def sample_algebra_element(self): return np.array([self.f.m(v) for v in self.ch.sample_ef()], dtype=np.uint32)
    def sample_bits(self, bits): return self.ch.sample_bits(bits)

    def grind(self, bits):
        if bits == 0:
            return 0
        for cand in range(BabyBear.P):                                 # serial semantics: the smallest witness
            c2 = copy.deepcopy(self.ch)
            c2.observe(cand)
            if c2.sample_bits(bits) == 0:
                self.ch = c2
                return self.f.m(cand)


def test_prove_driver_writes_the_fibonacci_fixture(monkeypatch):
    import fixture_replay as FR
    import mock_device as M
    import stark_verify as V
    from types import SimpleNamespace
    from oracle import p3_oracle as O
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.poseidon2 import Poseidon2
    from plonky3_b200.uni_stark import prove, verify
    from plonky3_b200.verifier import VerificationError

    class AirMockGpu(M.MockGpu):
        """The mock device answering the constraint-program entry points with the oracle."""

        def air_program_create(self, field, nodes, constraints, width, n_public):
            self._note("air_program_create")
            return (field, np.asarray(nodes, dtype=np.uint32), np.asarray(constraints, dtype=np.uint32))

        def air_quotient(self, prog, lde, log_q, log_n, public_values, alpha):
            self._note("air_quotient")
            field, nodes, cons = prog
            return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_q, log_n, list(public_values), M._n(alpha)))

    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    gold = json.loads((GOLD / "uni_stark_two_adic_v1.json").read_text())
    rc_i, rc_t, rc_p = FR.fixture_constants()
    gpu = AirMockGpu()
    pm = Poseidon2.new(BabyBear, 16, rc_i, rc_t, rc_p, monty=True)
    mmcs = MerkleTreeMmcs.poseidon2(pm, None, 0, gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(BabyBear, gpu), mmcs, FriParameters(2, 2, 1, 2, 1, 1, mmcs))     # fib_air.rs:134-155
    operm = O.make_perm(BabyBear.id, 16, rc_i, rc_t, rc_p, monty=True)
    config = SimpleNamespace(pcs=pcs, initialise_challenger=lambda: BabyBearChallenger(operm))
    air = SymbolicAir(BabyBear, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    trace = torch.from_numpy(E.fib_trace(BabyBear, 8).view(np.int32))
    proof = prove(config, air, trace, [0, 1, 21])
    raw = proof.to_postcard()
    assert len(raw) == 1115 and raw.hex() == gold["postcard_hex"]
    assert {"air_program_create", "air_quotient"} <= set(gpu.calls)
    _, _, cfg = None, None, dict(hasher=O.poseidon2_hasher(operm, operm), challenger_perm=operm, challenger_width=16, challenger_rate=8,
                                 log_blowup=2, log_final_poly_len=2, max_log_arity=1, num_queries=2, commit_pow_bits=1, query_pow_bits=1)
    verify(V.product_config(BabyBear, cfg), air, raw, [0, 1, 21])
    with pytest.raises(VerificationError):
        verify(V.product_config(BabyBear, cfg), air, raw, [0, 1, 22])
    # errors before anything runs
    gpu.calls.clear()
    with pytest.raises(ValueError, match="public values"):
        prove(config, air, trace, [0, 1])
    deg5 = SymbolicAir(BabyBear, 60, E.mul_air_eval(6, False, False), gpu=gpu)    # 8 chunks > blowup 4
    with pytest.raises(ValueError, match="quotient chunks"):
        prove(config, deg5, torch.from_numpy(E.mul_air_trace(BabyBear, 8, 6, False, False).view(np.int32)))
    assert gpu.calls == []
