"""The debug constraint check on the GPU (csrc/air_check.cu through air.check_constraints / check_all_constraints), over BabyBear and
KoalaBear: every example SymbolicAir and every hand-written AIR passes on its generated trace; single tampered cells give exactly
the oracle's failures (tests/test_air_check_cpu.py), check_constraints names the oracle's first failing row, and max_failures cuts
between rows; both passes write every count and nothing past the listed rows' ranges on poisoned buffers; heights beyond one sweep
of the persistent grid for a small and a large-slot program; `prove(check_constraints=True)`; bad arguments refused before any
launch."""
import ctypes as C
import importlib.util
import pathlib

import numpy as np
import pytest
import torch

import air_examples as E
from plonky3_b200 import _lib
from plonky3_b200.air import ConstraintViolation, MAIN_NEXT, SymbolicAir, check_all_constraints, check_constraints
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import StarkConfig, prove
from test_air_check_cpu import FIELDS, example_airs, oracle_failures, tamper

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
POISON = -1                                                            # 0xffffffff


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


def pairs(report):
    return [(f.row, f.constraint) for f in report.failures]


def capped(want, cap):
    """check_all_constraints' cap on the oracle's failures: rows are visited while fewer than `cap` failures are collected."""
    out = []
    for row in sorted({r for r, _ in want}):
        if cap is not None and len(out) >= cap:
            break
        out += [(r, k) for r, k in want if r == row]
    return out


def expect_all(air, trace_np, pis=(), caps=(None,)):
    """The device check of trace_np against the oracle: the full report, check_constraints, and each cap."""
    want = oracle_failures(air, trace_np, pis)
    t = dev(trace_np)
    rep = check_all_constraints(air, t, pis)
    assert pairs(rep) == want
    assert rep.total_rows == trace_np.shape[0] and rep.total_constraints_per_row == len(air.constraints)
    assert rep.is_ok() == (not want)
    if want:
        with pytest.raises(ConstraintViolation) as e:
            check_constraints(air, t, pis)
        row = want[0][0]
        assert e.value.row == row and [(f.row, f.constraint) for f in e.value.failures] == [p for p in want if p[0] == row]
        assert str(e.value).startswith(f"constraints not satisfied on row {row}: failed constraints = [#")
    else:
        check_constraints(air, t, pis)
    for cap in caps:
        assert pairs(check_all_constraints(air, t, pis, max_failures=cap)) == capped(want, cap), cap
    return want


# ---- the example AIRs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("n", [1, 2, 3, 8, 1000])
def test_example_airs(gpu, field, n):
    for name, air, trace, pis in example_airs(field, n, gpu):
        assert expect_all(air, trace, pis) == [], name
        for row in sorted({0, n // 2, n - 1}):
            for col in sorted({0, air.width() - 1}):
                expect_all(air, tamper(field, trace, row, col), pis)
        if n > 1:                                                      # a cell the previous row reads as its next row
            col = next((int(a) for op, a, _, _ in air.nodes if op == MAIN_NEXT), None)
            if col is not None:
                expect_all(air, tamper(field, trace, n - 1, col), pis)
    name, air, trace, pis = example_airs(field, n, gpu)[0]
    bad = list(pis); bad[2] = (bad[2] + 1) % field.P
    assert expect_all(air, trace, bad)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_max_failures_cuts_between_rows(gpu, field):
    n = 64
    air = example_airs(field, n, gpu)[1][1]                            # MulAir: 60 constraints per row
    rng = np.random.default_rng(11)
    bad = E.mul_air_trace(field, n)
    for row in (3, 4, 9, 40, 63):
        bad[row, rng.integers(0, air.width(), 5)] = rng.integers(0, field.P, 5)
    want = expect_all(air, bad, (), caps=(0, 1, 2, 3, 7, 60, 10 ** 6))
    assert len({r for r, _ in want}) >= 4


# ---- the hand-written AIRs -------------------------------------------------------------------------------------------------
def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


HAND = [("keccak", 5), ("blake3", 2), ("sha256", 2), ("poseidon1", 1), ("poseidon2", 1)]


def _hand(gpu, name, f, log_rows):
    make, _, hashes, random_inputs, dtype = _air_prove().AIRS[name]
    air = make(f, gpu)
    inputs = torch.from_numpy(np.ascontiguousarray(random_inputs(f, hashes(log_rows))).view(dtype)).cuda()
    return air, air.generate_trace_rows(inputs)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("name,log_rows", HAND, ids=[h[0] for h in HAND])
def test_hand_written_airs(gpu, field, name, log_rows):
    air, trace = _hand(gpu, name, field, log_rows)
    n_insns, n_slots, n_cons = air.check_program().info()
    assert n_cons == len(air.constraints)
    if name in ("keccak", "blake3", "sha256"):
        assert n_slots > 384
    t = host(trace)
    H = t.shape[0]
    assert check_all_constraints(air, trace).is_ok()
    rng = np.random.default_rng(5)
    cells = [(0, int(rng.integers(air.width()))), (H - 1, int(rng.integers(air.width()))), (H // 2, int(rng.integers(air.width())))]
    nxt = sorted({int(a) for op, a, _, _ in air.nodes if op == MAIN_NEXT})
    if nxt:
        cells.append((H // 2 + 1, nxt[len(nxt) // 2]))
    for row, col in cells:
        want = expect_all(air, tamper(field, t, row, col), caps=(1,))
        assert want, (row, col)


# ---- poisoned outputs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_poisoned_outputs(gpu, field):
    n = 1000
    air = example_airs(field, n, gpu)[1][1]
    bad = E.mul_air_trace(field, n)
    for row in (0, 17, 500, 999):
        bad[row, [1, 2, 4, 7]] += 1
    want = oracle_failures(air, bad)
    t = dev(bad)
    prog = air.check_program()
    counts = torch.full((n + 64,), POISON, dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_air_check_dev(gpu.h, prog.h, t.data_ptr(), n, None, None, 0, None, counts.data_ptr()))
    c = host(counts)
    assert (c[n:] == 0xFFFFFFFF).all() and (c[:n] < 0xFFFFFFFF).all()
    exp = np.zeros(n, dtype=np.uint32)
    for r, _ in want:
        exp[r] += 1
    assert np.array_equal(c[:n], exp)
    rows = [999, 17, 500]                                              # any order, ranges with gaps between them
    gap = 5
    offs, at = [], gap
    for r in rows:
        offs.append(at); at += int(exp[r]) + gap
    failed = torch.full((at,), POISON, dtype=torch.int32, device="cuda")
    d_rows = torch.tensor(rows, dtype=torch.int32, device="cuda")
    d_offs = torch.tensor(offs, dtype=torch.int64, device="cuda")
    _lib.check(gpu.L.p3gpu_air_check_rows_dev(gpu.h, prog.h, t.data_ptr(), n, None, None, 0, None, d_rows.data_ptr(), len(rows),
                                              d_offs.data_ptr(), failed.data_ptr()))
    got = host(failed)
    written = np.zeros(at, dtype=bool)
    for r, o in zip(rows, offs):
        assert got[o:o + exp[r]].tolist() == [k for rr, k in want if rr == r]
        written[o:o + exp[r]] = True
    assert (got[~written] == 0xFFFFFFFF).all()


# ---- beyond one sweep of the persistent grid ---------------------------------------------------------------------------------
@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_persistent_sweep_small_program(gpu, field):
    n = 1 << 20
    fib = E.fib_trace(field, n)
    pis = [0, 1, field.from_monty(int(fib[-1, 1]))]
    air = SymbolicAir(field, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    assert air.check_program().info()[1] * 128 * 4 * 132 * 16 < 1 << 30        # the grid is capped at 16 blocks per SM: 2^18 threads
    bad = tamper(field, fib, n - 3, 1)
    expect_all(air, bad, pis)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_persistent_sweep_large_program(gpu, field):
    log_rows = 17
    air, trace = _hand(gpu, "sha256", field, log_rows)
    slots = air.check_program().info()[1]
    assert (1 << log_rows) > 2 * ((1 << 30) // (slots * 128 * 4)) * 128      # rows beyond two sweeps of the grid the scratch bound allows
    assert check_all_constraints(air, trace).is_ok()
    H, row = 1 << log_rows, (1 << log_rows) - 7
    col = 4321
    trace[row, col] = int((int(trace[row, col]) + 1) % field.P)
    rep = check_all_constraints(air, trace)
    # rows are independent (no next row, no selectors): the oracle of the one tampered row
    want = [(row, k) for _, k in oracle_failures(air, host(trace[row:row + 1]))]
    assert want and pairs(rep) == want
    with pytest.raises(ConstraintViolation) as e:
        check_constraints(air, trace)
    assert e.value.row == row


# ---- prove(check_constraints=True) -----------------------------------------------------------------------------------------
def _config(gpu, field):
    p16, p24 = default_poseidon2(field, 16), default_poseidon2(field, 24)
    mmcs = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=2, gpu=gpu)
    return StarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), mmcs, FriParameters(2, 1, 3, 20, 0, 4, mmcs)), p24, 16)


@pytest.mark.parametrize("field", FIELDS, ids=lambda f: f.name)
def test_checking_prove(gpu, field, monkeypatch):
    n = 64
    config = _config(gpu, field)
    air = SymbolicAir(field, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    fib = E.fib_trace(field, n)
    pis = [0, 1, field.from_monty(int(fib[-1, 1]))]
    raw = prove(config, air, dev(fib), pis).to_postcard()
    assert prove(config, air, dev(fib), pis, check_constraints=True).to_postcard() == raw

    def no_commit(*a, **k):
        raise AssertionError("pcs.commit reached")
    monkeypatch.setattr(config.pcs, "commit", no_commit)
    with pytest.raises(ConstraintViolation, match="constraints not satisfied on row 40: failed constraints = \\[#2\\]$"):
        prove(config, air, dev(tamper(field, fib, 41, 0)), pis, check_constraints=True)


# ---- argument errors -------------------------------------------------------------------------------------------------------
def test_bad_arguments_are_refused_before_launch(gpu):
    from air_preprocessed_examples import mixed_air, mixed_trace
    f, n = KoalaBear, 16
    L = gpu.L
    air = mixed_air(f, n, gpu)                                         # preprocessed + periodic columns
    prog = air.check_program()
    t, pre = dev(mixed_trace(f, n)), dev(air.preprocessed_trace())
    per = dev(np.zeros((4, 2), dtype=np.uint32))
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    rows = torch.tensor([3, 16], dtype=torch.int32, device="cuda")
    offs = torch.tensor([0, 1], dtype=torch.int64, device="cuda")
    out = torch.zeros(8, dtype=torch.int32, device="cuda")
    fib = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    fprog = fib.check_program()
    bad_pub = np.array([0, 1, f.P], dtype=np.uint32)
    gpu._use_torch_stream()
    before = gpu.launches
    EINVAL = _lib.EINVAL
    p = lambda x: x.data_ptr()
    assert L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, p(counts)) == _lib.EOK
    before = gpu.launches
    cases = [
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, None, p(per), 4, None, p(counts)),                 # preprocessed missing
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, p(pre), None, 4, None, p(counts)),                 # periodic missing
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 0, None, p(counts)),                # no periodic rows
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), 0, p(pre), p(per), 4, None, p(counts)),                # height 0
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t) + 2, n, p(pre), p(per), 4, None, p(counts)),           # misaligned trace
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, p(pre) + 1, p(per), 4, None, p(counts)),           # misaligned preprocessed
        L.p3gpu_air_check_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, p(counts) + 2),           # misaligned counts
        L.p3gpu_air_check_dev(gpu.h, fprog.h, p(t), n, p(pre), None, 0, None, p(counts)),                # preprocessed given, undeclared
        L.p3gpu_air_check_dev(gpu.h, fprog.h, p(t), n, None, None, 0, None, p(counts)),                  # public values missing
        L.p3gpu_air_check_dev(gpu.h, fprog.h, p(t), n, None, None, 0, bad_pub.ctypes.data, p(counts)),   # non-canonical public value
        L.p3gpu_air_check_dev(gpu.h, air.program().h, p(t), n, p(pre), p(per), 4, None, p(counts)),      # a quotient program
        L.p3gpu_air_check_rows_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, p(rows), 2, p(offs), p(out)),  # row 16 >= 16
        L.p3gpu_air_check_rows_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, p(rows), 1, p(offs) + 4, p(out)),  # misaligned
        L.p3gpu_air_check_rows_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, None, 1, p(offs), p(out)),    # null rows
    ]
    assert cases == [EINVAL] * len(cases), cases
    assert gpu.launches == before
    # a check program is not a quotient program
    alpha = np.array([f.to_monty(v) for v in (3, 5, 7, 11)], dtype=np.uint32)
    lde = dev(np.zeros((2 * n, 2), dtype=np.uint32))
    q = torch.zeros((2 * n, 4), dtype=torch.int32, device="cuda")
    pv = np.array([0, 1, 1], dtype=np.uint32)
    assert L.p3gpu_air_quotient_dev(gpu.h, fprog.h, p(lde), 5, 5, 4, pv.ctypes.data, alpha.ctypes.data, p(q)) == EINVAL
    assert "p3gpu_air_check_program_create" in L.p3gpu_last_error().decode()
    assert L.p3gpu_air_quotient_layout_dev(gpu.h, prog.h, p(lde), 5, p(dev(np.zeros((2 * n, 1), dtype=np.uint32))), 5, p(per), 2, 5,
                                           4, None, alpha.ctypes.data, p(q)) == EINVAL
    assert gpu.launches == before
    n_insns, n_slots, n_cons = C.c_size_t(), C.c_size_t(), C.c_size_t()
    _lib.check(L.p3gpu_air_program_info(prog.h, C.byref(n_insns), C.byref(n_slots), C.byref(n_cons)))
    assert n_cons.value == 2 and n_insns.value > 0
    # an empty row list launches nothing
    _lib.check(L.p3gpu_air_check_rows_dev(gpu.h, prog.h, p(t), n, p(pre), p(per), 4, None, None, 0, None, None))
    assert gpu.launches == before
