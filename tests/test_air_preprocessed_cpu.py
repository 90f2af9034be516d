"""Preprocessed and periodic columns on the CPU: the compiler and the per-row semantics of csrc/air_program.cuh (run on the host by
tests/cpp/air_layout_check.cpp) against the oracle (tests/air_layout_oracle.py, which evaluates periodic columns directly, not through
the padded LDE table), the new leaves' validation, equivalences with the leaves they stand in for, the errors `prove` raises before any
device call, and proofs of MulFibPAir, PeriodicAir and an AIR with both kinds made by the product `prove` on the oracle-backed stand-in
device, accepted and rejected by the product verifier and by the restated verifier (tests/stark_verify_layout.py)."""
import os
import pathlib
import subprocess

import numpy as np
import pytest
import torch

import air_layout_oracle as AL
import air_oracle as A
import air_preprocessed_examples as X
import mock_device as M
from plonky3_b200 import _lib
from plonky3_b200.air import (ADD, CONST, IS_FIRST_ROW, IS_TRANSITION, MAIN_LOCAL, MAIN_NEXT, MUL, PERIODIC, PREPROCESSED_LOCAL,
                              PREPROCESSED_NEXT, PUBLIC, SUB, SymbolicAir)
from plonky3_b200.field import BabyBear, KoalaBear
from test_air_program_cpu import checker, _inputs  # noqa: F401  (module-scoped fixture)

ROOT = pathlib.Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def layout_checker(tmp_path_factory):
    exe = tmp_path_factory.mktemp("air_layout") / "air_layout_check"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "air_layout_check.cpp"), "-o", str(exe)],
                   check=True)
    return exe


class LayoutMockGpu(M.MockGpu):
    """The stand-in device answering the constraint-program entry points with the oracle (the periodic table as given)."""

    def air_program_create(self, field, nodes, constraints, width, n_public):
        self._note("air_program_create")
        return (field, np.asarray(nodes, dtype=np.uint32), np.asarray(constraints, dtype=np.uint32))

    def air_program_create_layout(self, field, nodes, constraints, layout):
        self._note("air_program_create_layout")
        return (field, np.asarray(nodes, dtype=np.uint32), np.asarray(constraints, dtype=np.uint32))

    def air_quotient(self, prog, lde, log_q, log_n, public_values, alpha):
        self._note("air_quotient")
        field, nodes, cons = prog
        return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_q, log_n, list(public_values), M._n(alpha)))

    def air_quotient_layout(self, prog, lde, pre_lde, periodic, log_q, log_n, public_values, alpha):
        self._note("air_quotient_layout")
        field, nodes, cons = prog
        return M._t(AL.air_quotient(field, nodes, cons, M._n(lde), log_q, log_n, list(public_values), M._n(alpha),
                                    pre_lde_bitrev=None if pre_lde is None else M._n(pre_lde),
                                    periodic_table=None if periodic is None else M._n(periodic)))


def _run(exe, job):
    out = subprocess.run([str(exe)], input=" ".join(map(str, job)), capture_output=True, text=True, check=True).stdout.split("\n")
    return tuple(int(v) for v in out[0].split()), out


def _layout_job(mode, field, layout, nodes, cons):
    nodes = np.asarray(nodes, dtype=np.uint32).reshape(-1, 4)
    cons = np.asarray(cons, dtype=np.uint32).ravel()
    return [mode, field.id, *layout, nodes.shape[0], cons.size, *nodes.ravel().tolist(), *cons.tolist()]


def run_compile_layout(exe, field, layout, nodes, cons):
    return _run(exe, _layout_job("L", field, layout, nodes, cons))[0]


def run_quotient_layout(exe, field, layout, nodes, cons, lde, pre, table, log_q, log_n, pubs, alpha):
    width, n_public, pre_width, n_periodic = layout
    table = np.zeros((1, 0), dtype=np.uint32) if table is None else np.asarray(table, dtype=np.uint32)
    pre = np.zeros((1 << log_q, 0), dtype=np.uint32) if pre is None else np.asarray(pre)
    log_rows = int(table.shape[0]).bit_length() - 1
    job = _layout_job("Q", field, layout, nodes, cons) + [log_q, log_n, *np.asarray(lde)[: 1 << log_q].ravel().tolist(),
                                                          *pre[: 1 << log_q].ravel().tolist(), log_rows, *table.ravel().tolist(),
                                                          *list(pubs), *np.asarray(alpha).tolist()]
    head, out = _run(exe, job)
    return head, np.array(out[1].split(), dtype=np.uint32).reshape(-1, 4)


def periodic_table(field, columns, log_n, log_q):
    """The table SymbolicAir builds (with the stand-in device's oracle LDE)."""
    air = SymbolicAir(field, 1, lambda b: None, periodic_columns=columns, gpu=LayoutMockGpu())
    return M._n(air.periodic_table(log_n, log_q))


def random_layout_dag(field, rng, width, n_public, pre_width, n_periodic, n_nodes, n_cons):
    """Leaves of every kind (preprocessed and periodic included), then operations on random earlier nodes."""
    kinds = [(MAIN_LOCAL, width), (MAIN_NEXT, width), (CONST, 0), (PUBLIC, n_public), (IS_FIRST_ROW, 0), (IS_TRANSITION, 0),
             (PREPROCESSED_LOCAL, pre_width), (PREPROCESSED_NEXT, pre_width), (PERIODIC, n_periodic)]
    nodes = []
    for op, bound in kinds:
        if op == CONST:
            nodes.append((CONST, 0, 0, field.to_monty(int(rng.integers(field.P)))))
        elif bound or op in (IS_FIRST_ROW, IS_TRANSITION):
            nodes.append((op, int(rng.integers(bound)) if bound else 0, 0, 0))
    while len(nodes) < n_nodes:
        i = len(nodes)
        op = int(rng.choice([ADD, SUB, MUL, PREPROCESSED_LOCAL, PERIODIC, PREPROCESSED_NEXT]))
        if op in (PREPROCESSED_LOCAL, PREPROCESSED_NEXT):
            nodes.append((op, int(rng.integers(pre_width)), 0, 0))
        elif op == PERIODIC:
            nodes.append((op, int(rng.integers(n_periodic)), 0, 0))
        else:
            nodes.append((op, int(rng.integers(i)), int(rng.integers(i)), 0))
    cons = [int(v) for v in rng.integers(0, n_nodes, n_cons)]
    return np.array(nodes, dtype=np.uint32), cons


def _pre(field, rng, rows, width):
    return field.to_monty_array(rng.integers(0, field.P, (rows, width)).astype(np.uint64)).astype(np.uint32)


def _periodic_columns(field, rng, periods):
    return [[int(v) for v in rng.integers(0, field.P, p)] for p in periods]


# ---------------------------------------------------------------- compiler + per-row semantics vs the oracle
# (width, n_public, pre_width, periods, n_nodes, n_cons, log_n, q)
SHAPES = [(3, 1, 2, [4, 2], 80, 8, 4, 1), (5, 0, 7, [1, 8, 16], 200, 20, 5, 2), (2, 2, 1, [32], 60, 5, 5, 0),
          (4, 1, 3, [2, 2, 64], 150, 12, 6, 3)]
CASES = [(f, k) for f in (BabyBear, KoalaBear) for k in range(len(SHAPES))]


@pytest.mark.parametrize("f,k", CASES, ids=[f"{c[0].name}-{c[1]}" for c in CASES])
def test_random_dags_with_every_leaf_kind_match_oracle(layout_checker, f, k):
    width, n_public, pre_width, periods, n_nodes, n_cons, log_n, q = SHAPES[k]
    rng = np.random.default_rng(100 + k)
    nodes, cons = random_layout_dag(f, rng, width, n_public, pre_width, len(periods), n_nodes, n_cons)
    log_q = log_n + q
    lde, pubs, alpha = _inputs(f, rng, width, n_public, log_q)
    pre = _pre(f, rng, 1 << log_q, pre_width)
    cols = _periodic_columns(f, rng, periods)
    table = periodic_table(f, cols, log_n, log_q)
    assert table.shape == (max(periods) << q, len(periods))
    layout = (width, n_public, pre_width, len(periods))
    (rc, n_insn, slots, live), got = run_quotient_layout(layout_checker, f, layout, nodes, cons, lde, pre, table, log_q, log_n, pubs, alpha)
    assert rc == 0 and slots == live
    exp = AL.air_quotient(f.id, nodes, cons, lde, log_q, log_n, pubs, alpha, pre_lde_bitrev=pre, periodic_columns=cols)
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"first differing row {bad[:1]}"


def test_layout_programs_without_new_leaves_match_the_plain_run(checker, layout_checker):
    """A layout program that reads none of the new leaves gives the plain instance's result."""
    f = KoalaBear
    rng = np.random.default_rng(5)
    from test_air_program_cpu import random_dag, run_quotient
    nodes, cons = random_dag(f, rng, 6, 1, 100, 10)
    lde, pubs, alpha = _inputs(f, rng, 6, 1, 5)
    _, plain = run_quotient(checker, f, 6, 1, nodes, cons, lde, 5, 4, pubs, alpha)
    (rc, *_), lay = run_quotient_layout(layout_checker, f, (6, 1, 2, 1), nodes, cons, lde, _pre(f, rng, 32, 2), periodic_table(f, [[1, 2]], 4, 5),
                                        5, 4, pubs, alpha)
    assert rc == 0 and np.array_equal(plain, lay)


# ---------------------------------------------------------------- validation
def test_new_leaves_are_validated(checker, layout_checker):
    f = BabyBear
    layout = (2, 0, 3, 2)
    ok = [(PREPROCESSED_LOCAL, 2, 0, 0), (PREPROCESSED_NEXT, 0, 0, 0), (PERIODIC, 1, 0, 0), (MUL, 0, 1, 0), (ADD, 3, 2, 0)]
    assert run_compile_layout(layout_checker, f, layout, ok, [4])[0] == 0
    for nodes in ([(PREPROCESSED_LOCAL, 3, 0, 0)], [(PREPROCESSED_NEXT, 5, 0, 0)], [(PERIODIC, 2, 0, 0)]):
        assert run_compile_layout(layout_checker, f, layout, nodes, [0])[0] == _lib.EINVAL, nodes
    for op in range(11, 16):                                            # still unknown node ops
        assert run_compile_layout(layout_checker, f, layout, [(MAIN_LOCAL, 0, 0, 0), (op, 0, 0, 0)], [1])[0] == _lib.EINVAL, op
    assert run_compile_layout(layout_checker, f, layout, [(19, 0, 0, 0)], [0])[0] == _lib.EINVAL
    # the layout-free entry point has no preprocessed or periodic columns
    from test_air_program_cpu import run_compile
    for nodes in ([(PREPROCESSED_LOCAL, 0, 0, 0)], [(PERIODIC, 0, 0, 0)]):
        assert run_compile(checker, f, 2, 0, nodes, [0])[0] == _lib.EINVAL


def test_symbolic_air_refuses_bad_declarations():
    f = BabyBear
    pre = np.zeros((8, 1), dtype=np.uint32)
    with pytest.raises(ValueError, match="preprocessed next row"):
        SymbolicAir(f, 1, lambda b: b.assert_zero(b.preprocessed().next[0]), preprocessed_trace=pre, preprocessed_next_row_columns=[])
    for cols in ([[1, 2, 3]], [[]], [[1, 2], [1] * 6]):
        with pytest.raises(ValueError, match="power of two"):
            SymbolicAir(f, 1, lambda b: None, periodic_columns=cols)
    with pytest.raises(IndexError):
        SymbolicAir(f, 1, lambda b: b.assert_zero(b.preprocessed().local[1]), preprocessed_trace=pre)
    air = SymbolicAir(f, 1, lambda b: b.assert_zero(b.preprocessed().local[0] * b.periodic_values()[0]), preprocessed_trace=pre,
                      periodic_columns=[[1, 2]])
    assert (air.preprocessed_width(), air.preprocessed_next_row_columns(), air.num_periodic_columns()) == (1, [0], 1)
    assert air.constraint_degrees() == [2]                              # degree_multiple 1 for both leaf kinds


# ---------------------------------------------------------------- equivalences (bit-identical quotient values)
def _quotient(exe, f, layout, nodes, cons, lde, pre, table, log_q, log_n, alpha):
    (rc, *_), q = run_quotient_layout(exe, f, layout, nodes, cons, lde, pre, table, log_q, log_n, [], alpha)
    assert rc == 0
    return q


@pytest.mark.parametrize("f", [BabyBear, KoalaBear])
def test_equivalent_leaves_give_identical_quotients(checker, layout_checker, f):
    rng = np.random.default_rng(9)
    log_n, q = 4, 2
    log_q = log_n + q
    lde, _, alpha = _inputs(f, rng, 3, 0, log_q)
    c = int(rng.integers(1, f.P))
    from test_air_program_cpu import run_quotient
    # a period-1 column == the constant
    with_const = [(MAIN_LOCAL, 0, 0, 0), (CONST, 0, 0, f.to_monty(c)), (MUL, 0, 1, 0), (MAIN_NEXT, 2, 0, 0), (SUB, 2, 3, 0)]
    with_per = [(MAIN_LOCAL, 0, 0, 0), (PERIODIC, 0, 0, 0), (MUL, 0, 1, 0), (MAIN_NEXT, 2, 0, 0), (SUB, 2, 3, 0)]
    _, want = run_quotient(checker, f, 3, 0, with_const, [4, 2], lde, log_q, log_n, [], alpha)
    got = _quotient(layout_checker, f, (3, 0, 0, 1), with_per, [4, 2], lde, None, periodic_table(f, [[c]], log_n, log_q), log_q, log_n, alpha)
    assert np.array_equal(got, want)
    # a preprocessed column equal to main column 1 == MAIN_LOCAL 1 / MAIN_NEXT 1
    main = [(MAIN_LOCAL, 1, 0, 0), (MAIN_NEXT, 1, 0, 0), (MAIN_LOCAL, 0, 0, 0), (MUL, 0, 2, 0), (SUB, 3, 1, 0), (IS_FIRST_ROW, 0, 0, 0),
            (MUL, 5, 0, 0)]
    prep = [(PREPROCESSED_LOCAL, 0, 0, 0), (PREPROCESSED_NEXT, 0, 0, 0)] + main[2:]
    _, want = run_quotient(checker, f, 3, 0, main, [4, 6], lde, log_q, log_n, [], alpha)
    got = _quotient(layout_checker, f, (3, 0, 1, 0), prep, [4, 6], lde, np.ascontiguousarray(lde[:, 1:2]), None, log_q, log_n, alpha)
    assert np.array_equal(got, want)
    # a period-n periodic column == a preprocessed column holding the same values
    vals = [int(v) for v in rng.integers(0, f.P, 1 << log_n)]
    from oracle import p3_oracle as O
    pre_lde = O.coset_lde_batch(f.id, f.to_monty_array(np.array(vals, dtype=np.uint64)).astype(np.uint32).reshape(-1, 1), q + 1,
                                f.generator, bitrev_out=True)
    body = [(MAIN_LOCAL, 0, 0, 0), (MUL, 0, 1, 0), (ADD, 2, 0, 0)]
    a = _quotient(layout_checker, f, (3, 0, 0, 1), [(PERIODIC, 0, 0, 0)] + body, [3], lde, None,
                  periodic_table(f, [vals], log_n, log_q), log_q, log_n, alpha)
    b = _quotient(layout_checker, f, (3, 0, 1, 0), [(PREPROCESSED_LOCAL, 0, 0, 0)] + body, [3], lde, pre_lde, None, log_q, log_n, alpha)
    assert np.array_equal(a, b)


# ---------------------------------------------------------------- the product prove on the stand-in device
def _config(gpu, fri, device_challenger=False):
    """The BabyBear configuration of the reference's Fibonacci fixture with FriParameters(*fri); the transcript on the host oracle,
    or with device_challenger on the GPU's DuplexChallenger (the same sponge)."""
    import fixture_replay as FR
    from types import SimpleNamespace
    from oracle import p3_oracle as O
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.poseidon2 import Poseidon2
    from test_air_program_cpu import BabyBearChallenger
    rc_i, rc_t, rc_p = FR.fixture_constants()
    pm = Poseidon2.new(BabyBear, 16, rc_i, rc_t, rc_p, monty=True)
    mmcs = MerkleTreeMmcs.poseidon2(pm, None, 0, gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(BabyBear, gpu), mmcs, FriParameters(*fri, mmcs))
    operm = O.make_perm(BabyBear.id, 16, rc_i, rc_t, rc_p, monty=True)
    if device_challenger:
        from plonky3_b200.uni_stark import StarkConfig
        config = StarkConfig(pcs, pm, 8)                                 # DuplexChallenger<_, _, 16, 8>
    else:
        config = SimpleNamespace(pcs=pcs, initialise_challenger=lambda: BabyBearChallenger(operm))
    cfg = dict(hasher=O.poseidon2_hasher(operm, operm), challenger_perm=operm, challenger_width=16, challenger_rate=8, log_blowup=fri[0],
               log_final_poly_len=fri[1], max_log_arity=fri[2], num_queries=fri[3], commit_pow_bits=fri[4], query_pow_bits=fri[5])
    return config, cfg


# name -> (log_n, FriParameters(log_blowup, log_final_poly_len, max_log_arity, num_queries, commit PoW, query PoW))
ROUND_TRIPS = {"mul_fib_pair": (4, (2, 1, 2, 6, 0, 1)), "periodic_air": (6, (2, 3, 2, 40, 0, 8)), "mixed": (5, (1, 1, 1, 6, 0, 1))}


def _air_and_trace(name, n, gpu, tamper_index=None):
    f = BabyBear
    if name == "mul_fib_pair":
        return X.mul_fib_pair_air(f, n, gpu, tamper_index), X.mul_fib_pair_trace(f, n)
    if name == "periodic_air":
        return X.periodic_air(f, gpu), X.periodic_air_trace(f, n)
    return X.mixed_air(f, n, gpu), X.mixed_trace(f, n)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32))


@pytest.mark.parametrize("name", list(ROUND_TRIPS))
def test_round_trip_on_the_stand_in_device(monkeypatch, name):
    import stark_verify as V
    import stark_verify_layout as VL
    from plonky3_b200.proof_io import proof_from_postcard
    from plonky3_b200.uni_stark import PreprocessedVerifierKey, prove, setup_preprocessed, verify
    from plonky3_b200.verifier import VerificationError
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    log_n, fri = ROUND_TRIPS[name]
    n = 1 << log_n
    gpu = LayoutMockGpu()
    config, cfg = _config(gpu, fri)
    air, trace = _air_and_trace(name, n, gpu)
    setup = setup_preprocessed(config, air, log_n)
    data, vk = setup if setup else (None, None)
    proof = prove(config, air, _t(trace), preprocessed=data)
    raw = proof.to_postcard()
    assert "air_quotient_layout" in gpu.calls and "air_quotient" not in gpu.calls
    p = proof_from_postcard(raw)
    assert (p["preprocessed_local"] is None) == (vk is None)
    if name == "mixed":
        assert len(proof.quotient_chunks) == 2 and proof.preprocessed_next is None and p["preprocessed_next"] is None
    if name == "mul_fib_pair":
        assert proof.preprocessed_next is not None and len(proof.quotient_chunks) == 2      # is_transition has degree 0
    fld = V.Fld(BabyBear.id)
    sv_air = X.stark_verify_air(name)
    sv_vk = None if vk is None else {"width": vk.width, "degree_bits": vk.degree_bits, "commitment": vk.commitment}
    product = V.product_config(BabyBear, cfg)
    verify(product, air, raw, preprocessed_vk=vk)
    VL.verify(fld, cfg, sv_air, p, preprocessed_vk=sv_vk)

    def rejected(raw_or_proof, key=vk, sv_key=sv_vk, the_air=air):
        with pytest.raises(VerificationError):
            verify(product, the_air, raw_or_proof, preprocessed_vk=key)
        with pytest.raises(V.VerifyError):
            VL.verify(fld, cfg, sv_air, proof_from_postcard(raw_or_proof), preprocessed_vk=sv_key)

    if vk is not None:
        import copy                                                     # a changed preprocessed opened value
        bad = copy.deepcopy(proof)
        bad.preprocessed_local = np.array(bad.preprocessed_local, dtype=np.uint32)
        bad.preprocessed_local[0, 0] = (int(bad.preprocessed_local[0, 0]) + 1) % BabyBear.P
        rejected(bad.to_postcard())
        cap = np.array(vk.commitment, dtype=np.uint32).copy(); cap[0, 0] ^= 1                       # wrong commitment
        rejected(raw, PreprocessedVerifierKey(vk.width, vk.degree_bits, cap), dict(sv_vk, commitment=cap))
        rejected(raw, PreprocessedVerifierKey(vk.width + 1, vk.degree_bits, vk.commitment), dict(sv_vk, width=vk.width + 1))  # wrong width
        with pytest.raises(VerificationError):                                                      # no key at all
            verify(product, air, raw)
    if name == "mul_fib_pair":                                          # test_tampered_preprocessed_fails
        tampered, _ = _air_and_trace(name, n, gpu, tamper_index=3)
        _, tvk = setup_preprocessed(config, tampered, log_n)
        assert not np.array_equal(tvk.commitment, vk.commitment)
        rejected(raw, tvk, {"width": tvk.width, "degree_bits": tvk.degree_bits, "commitment": tvk.commitment})
    if name in ("periodic_air", "mixed"):                               # a trace that breaks a periodic constraint
        bad_trace = trace.copy()
        bad_trace[1, 0 if name == "periodic_air" else 1] ^= 1
        rejected(prove(config, air, _t(bad_trace), preprocessed=data).to_postcard())


def test_product_verifier_rejects_malformed_periods(monkeypatch):
    """An AIR object whose periods are 0, 3 or larger than the trace: VerificationError, not a crash (periodic_column_shape.rs)."""
    from plonky3_b200.uni_stark import prove
    from plonky3_b200.verifier import VerificationError, verify
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    log_n, fri = ROUND_TRIPS["periodic_air"]
    gpu = LayoutMockGpu()
    config, cfg = _config(gpu, fri)
    air = X.periodic_air(BabyBear, gpu)
    raw = prove(config, air, _t(X.periodic_air_trace(BabyBear, 1 << log_n))).to_postcard()
    import stark_verify as V
    product = V.product_config(BabyBear, cfg)
    for cols in ([[], [10, 20]], [[1, 2, 3], [10, 20]], [[1] * (2 << log_n), [10, 20]]):
        class Malformed:
            width, num_public_values, main_next_row_columns = air.width, air.num_public_values, air.main_next_row_columns
            max_constraint_degree, eval_folded_constraints = air.max_constraint_degree, air.eval_folded_constraints

            def periodic_columns(self, c=cols): return c
        with pytest.raises(VerificationError, match="periodic"):
            verify(product, Malformed(), raw)


def test_errors_before_any_device_call(monkeypatch):
    from plonky3_b200.uni_stark import PreprocessedProverData, prove, setup_preprocessed
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    gpu = LayoutMockGpu()
    config, _ = _config(gpu, (2, 1, 2, 6, 0, 1))
    air, trace = _air_and_trace("mul_fib_pair", 16, gpu)
    gpu.calls.clear()
    with pytest.raises(ValueError, match="setup_preprocessed"):                 # preprocessed columns, no prover data
        prove(config, air, _t(trace))
    data8 = PreprocessedProverData(2, 3, np.zeros((1, 8), dtype=np.uint32), None)
    with pytest.raises(ValueError, match="height"):                             # prover data of another height
        prove(config, air, _t(trace), preprocessed=data8)
    with pytest.raises(ValueError, match="width"):                              # prover data of another width
        prove(config, air, _t(trace), preprocessed=PreprocessedProverData(3, 4, np.zeros((1, 8), dtype=np.uint32), None))
    with pytest.raises(ValueError, match="height"):                             # setup for a height the preprocessed trace lacks
        setup_preprocessed(config, air, 5)
    per = X.periodic_air(BabyBear, gpu, columns=[[1] * 32, [10, 20]])
    with pytest.raises(ValueError, match="exceeds the trace length"):           # period > n
        prove(config, per, _t(X.periodic_air_trace(BabyBear, 16, [[1] * 32, [10, 20]])))
    with pytest.raises(ValueError, match="width"):                              # prover data for an AIR without preprocessed columns
        prove(config, per, _t(X.periodic_air_trace(BabyBear, 16)), preprocessed=data8)
    assert gpu.calls == []


def test_proofs_without_the_new_columns_keep_their_bytes():
    from plonky3_b200.proof_io import proof_from_postcard
    import json
    import pathlib
    raw = bytes.fromhex(json.loads((pathlib.Path(__file__).resolve().parent / "golden" / "uni_stark_two_adic_v1.json").read_text())["postcard_hex"])
    p = proof_from_postcard(raw)
    assert p["preprocessed_local"] is None and p["preprocessed_next"] is None
