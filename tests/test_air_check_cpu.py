"""The debug constraint check on the CPU: the per-row check semantics of csrc/air_program.cuh (air_row_check, run on the host by
tests/cpp/air_check_host.cpp) against an independent numpy oracle on every failing (row, constraint), the check compiler's limits
next to the quotient compiler's unchanged ones, named assertions, the report types' wording, and `prove(check_constraints=True)`
refusing a sharded trace before any device call.

`constraint_values` / `oracle_failures` are the oracle the GPU tests (tests/test_gpu_air_check.py) compare against too: the
constraint DAG evaluated row by row with numpy, with the main-trace leaves of keccak_air_oracle.constraint_values plus public,
preprocessed and periodic leaves."""
import os
import pathlib
import subprocess

import numpy as np
import pytest

import air_examples as E
import air_preprocessed_examples as PE
from plonky3_b200 import _lib
from plonky3_b200.air import (ADD, CONST, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, MAIN_LOCAL, MAIN_NEXT, MUL, NEG, PERIODIC,
                              PREPROCESSED_LOCAL, PREPROCESSED_NEXT, PUBLIC, SUB, ConstraintFailure, ConstraintReport,
                              ConstraintViolation, SymbolicAir)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.uni_stark import StarkConfig, prove
from test_sharded_airs_cpu import Untouchable

ROOT = pathlib.Path(__file__).resolve().parent.parent
FIELDS = [BabyBear, KoalaBear]


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def _canon(field, m):
    rinv = pow(1 << 32, field.P - 2, field.P)
    return np.asarray(m, dtype=np.uint32).astype(np.int64) * rinv % field.P


def constraint_values(field, nodes, constraints, trace, public_values=(), preprocessed=None, periodic=()):
    """(K, H) int64: constraint k at row i, canonical.  trace / preprocessed: Montgomery (H, w) matrices; public_values: canonical;
    periodic: columns of canonical values, column k at row i is periodic[k][i mod len]."""
    p = field.P
    t = _canon(field, trace)
    H = t.shape[0]
    pre = _canon(field, preprocessed) if preprocessed is not None else None
    first = np.zeros(H, dtype=np.int64); first[0] = 1
    last = np.zeros(H, dtype=np.int64); last[-1] = 1
    sel = {IS_FIRST_ROW: first, IS_LAST_ROW: last, IS_TRANSITION: 1 - last}
    rows = np.arange(H)
    vals = []
    for op, a, b, imm in np.asarray(nodes, dtype=np.int64):
        if op == CONST:
            v = np.full(H, int(imm) * pow(1 << 32, p - 2, p) % p, dtype=np.int64)
        elif op == MAIN_LOCAL:
            v = t[:, a]
        elif op == MAIN_NEXT:
            v = np.roll(t[:, a], -1)
        elif op == PUBLIC:
            v = np.full(H, int(public_values[a]) % p, dtype=np.int64)
        elif op == PREPROCESSED_LOCAL:
            v = pre[:, a]
        elif op == PREPROCESSED_NEXT:
            v = np.roll(pre[:, a], -1)
        elif op == PERIODIC:
            col = np.array([int(x) % p for x in periodic[a]], dtype=np.int64)
            v = col[rows % len(col)]
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
    return np.stack([vals[int(k)] for k in constraints]) if len(constraints) else np.zeros((0, H), dtype=np.int64)


def oracle_failures(air, trace, public_values=()):
    """Every failing (row, constraint) of `air` on the Montgomery `trace`, rows ascending, constraints ascending within a row."""
    pre = air.preprocessed_trace()
    if pre is not None and not isinstance(pre, np.ndarray):
        pre = pre.cpu().numpy().view(np.uint32)
    v = constraint_values(air.field, air.nodes, air.constraints, trace, public_values, pre, air.periodic_columns())
    k, r = np.nonzero(v)
    return sorted(zip(r.tolist(), k.tolist()))


# ---- the host harness --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = tmp_path_factory.mktemp("air_check") / "air_check_host"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "air_check_host.cpp"), "-o", str(exe)],
                   check=True)
    return exe


def _head(mode, field, layout, nodes, cons):
    nodes = np.asarray(nodes, dtype=np.uint32).reshape(-1, 4)
    cons = np.asarray(cons, dtype=np.uint32).ravel()
    return [mode, field.id, *layout, nodes.shape[0], cons.size, *nodes.ravel().tolist(), *cons.tolist()]


def run_compile(exe, mode, field, layout, nodes, cons):
    """(rc, instructions, slots, message) of compiling under the check limits (mode C) or the quotient limits (mode P)."""
    r = subprocess.run([str(exe)], input=" ".join(map(str, _head(mode, field, layout, nodes, cons))), capture_output=True, text=True,
                       check=True)
    rc, n_insns, n_slots = (int(v) for v in r.stdout.split()[:3])
    return rc, n_insns, n_slots, r.stderr.strip()


def _layout(air):
    return (air.width(), air.num_public_values(), air.preprocessed_width(), air.num_periodic_columns())


def run_check(exe, air, trace, public_values=()):
    """The failing (row, constraint) pairs air_row_check reports on every row of `trace`."""
    f = air.field
    pre = air.preprocessed_trace()
    cols = air.periodic_columns()
    p_max = max((len(c) for c in cols), default=0)
    table = [f.to_monty(c[i % len(c)]) for i in range(p_max) for c in cols]
    job = _head("R", f, _layout(air), air.nodes, air.constraints) + [trace.shape[0], *np.asarray(trace).ravel().tolist(),
                                                                      *(np.asarray(pre).ravel().tolist() if pre is not None else []),
                                                                      p_max, *table, *[f.to_monty(int(v) % f.P) for v in public_values]]
    out = subprocess.run([str(exe)], input=" ".join(map(str, job)), capture_output=True, text=True, check=True).stdout.split("\n")
    assert int(out[0].split()[0]) == 0, out[0]
    pairs = [int(v) for v in out[1].split()]
    return list(zip(pairs[0::2], pairs[1::2]))


# ---- the example AIRs and their cases ----------------------------------------------------------------------------------------
MUL_VARIANTS = [(3, True, True), (2, True, True), (4, True, True), (3, False, True), (3, True, False), (3, False, False)]


def example_airs(field, n, gpu=None):
    """(name, air, valid trace, public values) of every example SymbolicAir at height n."""
    fib = E.fib_trace(field, n)
    out = [("fib", SymbolicAir(field, 2, E.fib_eval, num_public_values=3, gpu=gpu), fib,
            [0, 1, field.from_monty(int(fib[-1, 1]))])]
    for d, bnd, tr in MUL_VARIANTS:
        out.append((f"mul-{d}-{int(bnd)}{int(tr)}", SymbolicAir(field, 3 * E.REPETITIONS, E.mul_air_eval(d, bnd, tr), gpu=gpu),
                    E.mul_air_trace(field, n, d, bnd, tr), []))
    out.append(("mul_fib_pair", PE.mul_fib_pair_air(field, n, gpu=gpu), PE.mul_fib_pair_trace(field, n), []))
    out.append(("periodic_air", PE.periodic_air(field, gpu=gpu), PE.periodic_air_trace(field, n), []))
    out.append(("mixed", PE.mixed_air(field, n, gpu=gpu), PE.mixed_trace(field, n), []))
    return out


def tamper(field, trace, row, col):
    """`trace` with cell (row, col) moved to another canonical Montgomery word."""
    t = np.array(trace, dtype=np.uint32, copy=True)
    t[row, col] = (int(t[row, col]) + 1) % field.P
    return t


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("n", [1, 2, 3, 8, 1000])
def test_per_row_semantics_match_the_oracle(checker, field, n):
    for name, air, trace, pis in example_airs(field, n):
        assert oracle_failures(air, trace, pis) == [], name
        assert run_check(checker, air, trace, pis) == [], name
        rows = sorted({0, n - 1, n // 2})
        for row in rows:
            for col in sorted({0, air.width() - 1}):
                bad = tamper(field, trace, row, col)
                want = oracle_failures(air, bad, pis)
                assert run_check(checker, air, bad, pis) == want, (name, row, col)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("n", [1, 2, 3, 1000])
def test_wrong_public_values_and_preprocessed_cells(checker, field, n):
    name, air, trace, pis = example_airs(field, n)[0]
    for k in range(3):
        bad = list(pis)
        bad[k] = (bad[k] + 1) % field.P
        want = oracle_failures(air, trace, bad)
        assert want and run_check(checker, air, trace, bad) == want, k
    for row in sorted({0, n // 2, n - 1}):
        for air in (PE.mul_fib_pair_air(field, n, tamper_index=row), ):
            want = oracle_failures(air, PE.mul_fib_pair_trace(field, n))
            assert run_check(checker, air, PE.mul_fib_pair_trace(field, n)) == want, row
            if 0 < row < n - 1:                                     # row 0 has a = 0, which hides its product coefficient
                assert want, row
        mixed = PE.mixed_air(field, n)
        mixed._pre_trace = tamper(field, mixed.preprocessed_trace(), row, 0)
        want = oracle_failures(mixed, PE.mixed_trace(field, n))
        assert want and run_check(checker, mixed, PE.mixed_trace(field, n)) == want, row


# ---- the compiler's limits ---------------------------------------------------------------------------------------------------
def many_live(n):
    """A DAG whose program keeps n leaves live at once: constraint 0 sums n columns, constraints 1..n read each column again."""
    nodes = [(MAIN_LOCAL, c, 0, 0) for c in range(n)]
    acc = 0
    for c in range(1, n):
        nodes.append((ADD, acc, c, 0))
        acc = len(nodes) - 1
    return nodes, [acc] + list(range(n))


def test_a_check_program_has_no_constraint_or_384_slot_limit(checker):
    n = 3000
    nodes, cons = many_live(n)
    rc, n_insns, n_slots, _ = run_compile(checker, "C", KoalaBear, (n, 0, 0, 0), nodes, cons)
    assert rc == 0 and n_slots > 384 and len(cons) > 2048 and n_insns == len(nodes) + len(cons)
    air = SymbolicAir(KoalaBear, n, lambda b: None)
    air.nodes, air.constraints = np.array(nodes, dtype=np.uint32), np.array(cons, dtype=np.uint32)
    rng = np.random.default_rng(3)
    trace = np.zeros((3, n), dtype=np.uint32)
    trace[1] = rng.integers(1, KoalaBear.P, n)
    trace[2, ::7] = rng.integers(1, KoalaBear.P, trace[2, ::7].size)
    want = oracle_failures(air, trace)
    assert len(want) > 2048 and run_check(checker, air, trace) == want


def test_a_check_program_stops_at_the_16_bit_operand_field(checker):
    nodes, cons = many_live(65536)
    rc, _, _, msg = run_compile(checker, "C", BabyBear, (65536, 0, 0, 0), nodes, cons)
    assert rc == _lib.EUNSUPPORTED and msg == "AIR program: more than 65535 simultaneously live values (slots)"
    nodes, cons = many_live(65534)
    rc, _, n_slots, _ = run_compile(checker, "C", BabyBear, (65534, 0, 0, 0), nodes, cons)
    assert rc == 0 and n_slots == 65535


def test_the_quotient_compiler_keeps_its_limits_and_messages(checker):
    nodes, cons = many_live(385)
    rc, _, _, msg = run_compile(checker, "P", KoalaBear, (385, 0, 0, 0), nodes, cons)
    assert rc == _lib.EUNSUPPORTED and msg == "AIR program: more than 384 simultaneously live values (slots)"
    nodes = [(MAIN_LOCAL, 0, 0, 0)]
    rc, _, _, msg = run_compile(checker, "P", KoalaBear, (1, 0, 0, 0), nodes, [0] * 2049)
    assert rc == _lib.EUNSUPPORTED and msg == "AIR program: 2049 constraints (at most 2048)"
    assert run_compile(checker, "P", KoalaBear, (1, 0, 0, 0), nodes, [0] * 2048)[0] == 0
    assert run_compile(checker, "C", KoalaBear, (1, 0, 0, 0), nodes, [0] * 2049)[0] == 0


def test_the_check_compiler_validates_as_the_quotient_compiler(checker):
    bad = [([(MAIN_LOCAL, 2, 0, 0)], [0]), ([(PUBLIC, 0, 0, 0)], [0]), ([(ADD, 0, 0, 0)], [0]), ([(MAIN_LOCAL, 0, 0, 0)], [1]),
           ([(11, 0, 0, 0)], [0]), ([(CONST, 0, 0, KoalaBear.P)], [0]), ([(PREPROCESSED_LOCAL, 0, 0, 0)], [0]),
           ([(PERIODIC, 0, 0, 0)], [0])]
    for nodes, cons in bad:
        c = run_compile(checker, "C", KoalaBear, (2, 0, 0, 0), nodes, cons)
        q = run_compile(checker, "P", KoalaBear, (2, 0, 0, 0), nodes, cons)
        assert c[0] == _lib.EINVAL and c == q, (nodes, c, q)


# ---- named assertions --------------------------------------------------------------------------------------------------------
def _fib_named(b):
    m, pis = b.main(), b.public_values()
    l, r, nl, nr = m.local[0], m.local[1], m.next[0], m.next[1]
    b.when_first_row().assert_eq_named(l, pis[0], "first left")
    b.when_first_row().assert_eq(r, pis[1])
    t = b.when_transition()
    t.assert_eq_named(r, nl, "left is previous right")
    t.assert_zero_named(l + r - nr, "fibonacci step")
    b.when_last_row().assert_eq(r, pis[2])
    b.assert_one_named(l * 0 + 1, "one")
    b.assert_bool_named(l * 0, "bool")


def _fib_plain(b):
    m, pis = b.main(), b.public_values()
    l, r, nl, nr = m.local[0], m.local[1], m.next[0], m.next[1]
    b.when_first_row().assert_eq(l, pis[0])
    b.when_first_row().assert_eq(r, pis[1])
    t = b.when_transition()
    t.assert_eq(r, nl)
    t.assert_zero(l + r - nr)
    b.when_last_row().assert_eq(r, pis[2])
    b.assert_one(l * 0 + 1)
    b.assert_bool(l * 0)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_named_assertions_record_labels_and_change_nothing_else(checker, field):
    named, plain = SymbolicAir(field, 2, _fib_named, num_public_values=3), SymbolicAir(field, 2, _fib_plain, num_public_values=3)
    assert named.builder.labels == {0: "first left", 2: "left is previous right", 3: "fibonacci step", 5: "one", 6: "bool"}
    assert [named.constraint_label(k) for k in range(7)] == ["first left", None, "left is previous right", "fibonacci step", None,
                                                             "one", "bool"]
    assert plain.builder.labels == {}
    assert np.array_equal(named.nodes, plain.nodes) and np.array_equal(named.constraints, plain.constraints)
    assert named.constraint_degrees() == plain.constraint_degrees()
    from plonky3_b200.verifier import Ext
    e = Ext(field)
    rng = np.random.default_rng(7)
    r = lambda: [int(v) for v in rng.integers(0, field.P, 4)]
    args = ([r(), r()], [r(), r()], [1, 2, 3], r(), r(), r(), r())
    assert named.eval_folded_constraints(e, *args) == plain.eval_folded_constraints(e, *args)
    trace = tamper(field, E.fib_trace(field, 8), 3, 1)
    pis = [0, 1, field.from_monty(int(E.fib_trace(field, 8)[-1, 1]))]
    assert run_check(checker, named, trace, pis) == run_check(checker, plain, trace, pis) == oracle_failures(plain, trace, pis)


def test_report_wording_follows_the_reference():
    assert str(ConstraintFailure(4, 3)) == "#3"
    assert str(ConstraintFailure(4, 7, "carry")) == '#7 "carry"'
    assert str(ConstraintFailure(4, 7, 'say "hi"')) == '#7 "say \\"hi\\""'
    v = ConstraintViolation(4, [ConstraintFailure(4, 3), ConstraintFailure(4, 7)])
    assert isinstance(v, ValueError) and v.row == 4 and len(v.failures) == 2
    assert str(v) == "constraints not satisfied on row 4: failed constraints = [#3, #7]"
    assert ConstraintReport([], 8, 5).is_ok() and not ConstraintReport([ConstraintFailure(0, 0)], 8, 5).is_ok()


def test_checking_prove_refuses_a_sharded_trace_before_any_device_call():
    air = SymbolicAir(KoalaBear, 2, E.fib_eval, num_public_values=3)
    with pytest.raises(ValueError, match="check_constraints needs whole trace rows"):
        prove(StarkConfig(Untouchable(), None), air, Untouchable(), [0, 1, 2], shard=Untouchable(), check_constraints=True)


def test_the_check_needs_a_device():
    air = SymbolicAir(KoalaBear, 2, E.fib_eval, num_public_values=3)
    from plonky3_b200.air import check_all_constraints
    with pytest.raises(_lib.P3GpuError, match="no CPU fallback"):
        check_all_constraints(air, Untouchable(), [0, 1, 2])
