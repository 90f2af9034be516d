"""Any AIR as symbolic constraints: a builder that mirrors the reference's `AirBuilder` / `SymbolicAirBuilder`
(air/src/air.rs, air/src/symbolic/{builder,expression}.rs) and `SymbolicAir`, which gives `uni_stark.prove` / `verify` everything they
read from an AIR.

    def fib(b):                                   # uni-stark/tests/fib_air.rs:33-75
        m, pis = b.main(), b.public_values()
        l, r, nl, nr = m.local[0], m.local[1], m.next[0], m.next[1]
        b.when_first_row().assert_eq(l, pis[0]); b.when_first_row().assert_eq(r, pis[1])
        t = b.when_transition(); t.assert_eq(r, nl); t.assert_eq(l + r, nr)
        b.when_last_row().assert_eq(r, pis[2])
    air = SymbolicAir(BabyBear, 2, fib, num_public_values=3, gpu=gpu)

`eval` runs once, on the host, and records an expression DAG: identical subexpressions are one node (hash-consed), and every node
carries the reference's `degree_multiple` (expression.rs:44-48).  The prover compiles the DAG into a register program on the device
(p3gpu_air_program_create) and evaluates the quotient there (p3gpu_air_quotient_dev); there is no CPU evaluation of the quotient.
The verifier's constraint folder evaluates the same DAG at the out-of-domain point.

Preprocessed columns (`preprocessed_trace=`, read as `b.preprocessed().local[c]` / `.next[c]`) are committed once by
`uni_stark.setup_preprocessed`; periodic columns (`periodic_columns=[[v0, .., v_{p-1}], ..]`, read as `b.periodic_values()[k]`,
each period a power of two) are evaluated on the quotient domain from a small table the AIR builds on the device
(`periodic_table`, fri/src/periodic.rs).

`check_constraints` / `check_all_constraints` (air/src/check_constraints.rs:429-627) evaluate every constraint on every row of a
trace on the device, with the reference's debug semantics over the trace domain, and name the failing rows and constraints;
`uni_stark.prove(..., check_constraints=True)` runs the first before committing.  Assertions may carry labels
(`assert_zero_named`, air/src/named.rs), which the reports show.

Not offered: extension-field constraints (assert_zero_ext), ZK.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib
from .field import Field

# node ops (include/p3gpu.h P3GPU_AIR_*)
CONST, MAIN_LOCAL, MAIN_NEXT, PUBLIC, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, ADD, SUB, NEG, MUL = range(11)
PREPROCESSED_LOCAL, PREPROCESSED_NEXT, PERIODIC = 16, 17, 18
BINARY = (ADD, SUB, MUL)


class Expr:
    """A node of the expression DAG.  +, -, * and unary - with other expressions or Python integers; `x ** k` by squaring."""
    __slots__ = ("g", "i")

    def __init__(self, g: "SymbolicAirBuilder", i: int):
        self.g, self.i = g, i

    def _e(self, x) -> "Expr":
        return x if isinstance(x, Expr) else self.g.constant(x)

    def __add__(self, o): return self.g._node(ADD, self.i, self._e(o).i)
    def __radd__(self, o): return self.g._node(ADD, self._e(o).i, self.i)
    def __sub__(self, o): return self.g._node(SUB, self.i, self._e(o).i)
    def __rsub__(self, o): return self.g._node(SUB, self._e(o).i, self.i)
    def __mul__(self, o): return self.g._node(MUL, self.i, self._e(o).i)
    def __rmul__(self, o): return self.g._node(MUL, self._e(o).i, self.i)
    def __neg__(self): return self.g._node(NEG, self.i)

    def __pow__(self, e: int):
        """exp_u64: square and multiply (e >= 1)."""
        if e < 1:
            return self.g.constant(1)
        acc, base = None, self
        while e:
            if e & 1:
                acc = base if acc is None else acc * base
            e >>= 1
            if e:
                base = base * base
        return acc

    def degree(self) -> int:
        return self.g.degrees[self.i]


class _Row:
    def __init__(self, g, op, width, what="the trace width"):
        self.g, self.op, self.width, self.what = g, op, width, what

    def __len__(self): return self.width

    def __getitem__(self, c):
        if isinstance(c, slice):
            return [self[k] for k in range(*c.indices(self.width))]
        if not 0 <= c < self.width:
            raise IndexError(f"column {c} outside {self.what} {self.width}")
        return self.g._node(self.op, c)


class _Main:
    """builder.main(): `local[c]` (current row) and `next[c]` (next row)."""

    def __init__(self, g, width):
        self.local, self.next = _Row(g, MAIN_LOCAL, width), _Row(g, MAIN_NEXT, width)


class _Preprocessed:
    """builder.preprocessed(): `local[c]` (current row) and `next[c]` (next row) of the preprocessed trace."""

    def __init__(self, g, width):
        self.local = _Row(g, PREPROCESSED_LOCAL, width, "the preprocessed width")
        self.next = _Row(g, PREPROCESSED_NEXT, width, "the preprocessed width")


class _Ops:
    """AirBuilder's provided methods (air/src/air.rs) on top of assert_zero."""

    def assert_zero(self, x):
        raise NotImplementedError

    def assert_eq(self, x, y): self.assert_zero(self._root._e(x) - y)
    def assert_one(self, x): self.assert_zero(self._root._e(x) - 1)

    def assert_bool(self, x):
        x = self._root._e(x)
        self.assert_zero(x * (x - 1))

    # NamedAirBuilder (air/src/named.rs:127-190): the same constraint, with a label kept as host metadata for the check's reports
    def assert_zero_named(self, x, name):
        k = len(self._root.constraints)
        self.assert_zero(x)
        self._root.labels[k] = str(name)

    def assert_eq_named(self, x, y, name): self.assert_zero_named(self._root._e(x) - y, name)
    def assert_one_named(self, x, name): self.assert_zero_named(self._root._e(x) - 1, name)

    def assert_bool_named(self, x, name):
        x = self._root._e(x)
        self.assert_zero_named(x * (x - 1), name)

    def when(self, cond): return _Filtered(self, self._root._e(cond))
    def when_first_row(self): return self.when(self._root.is_first_row())
    def when_last_row(self): return self.when(self._root.is_last_row())
    def when_transition(self): return self.when(self._root.is_transition())

    def main(self): return self._root.main()
    def preprocessed(self): return self._root.preprocessed()
    def periodic_values(self): return self._root.periodic_values()
    def public_values(self): return self._root.public_values()
    def is_first_row(self): return self._root.is_first_row()
    def is_last_row(self): return self._root.is_last_row()
    def is_transition(self): return self._root.is_transition()


class _Filtered(_Ops):
    """FilteredAirBuilder: every assertion is multiplied by the condition."""

    def __init__(self, inner, cond: Expr):
        self._inner, self._cond, self._root = inner, cond, inner._root

    def assert_zero(self, x): self._inner.assert_zero(self._cond * self._root._e(x))


class SymbolicAirBuilder(_Ops):
    """Records an AIR's constraints as a hash-consed expression DAG (nodes in topological order)."""

    def __init__(self, field: Field, width: int, num_public_values: int = 0, preprocessed_width: int = 0, num_periodic: int = 0):
        self.field, self.width, self.num_public = field, int(width), int(num_public_values)
        self.preprocessed_width, self.num_periodic = int(preprocessed_width), int(num_periodic)
        self._root = self
        self.nodes: list = []          # (op, a, b, imm)
        self.degrees: list = []
        self.constraints: list = []    # node indices in assertion order
        self.labels: dict = {}         # constraint index -> label of a named assertion
        self._memo: dict = {}

    def _e(self, x) -> Expr:
        return x if isinstance(x, Expr) else self.constant(x)

    def _node(self, op, a=0, b=0, imm=0) -> Expr:
        key = (op, a, b, imm)
        i = self._memo.get(key)
        if i is None:
            d = self.degrees
            deg = {MAIN_LOCAL: 1, MAIN_NEXT: 1, IS_FIRST_ROW: 1, IS_LAST_ROW: 1, PREPROCESSED_LOCAL: 1, PREPROCESSED_NEXT: 1,
                   PERIODIC: 1}.get(op, 0)                                                          # degree_multiple
            if op in (ADD, SUB):
                deg = max(d[a], d[b])
            elif op == NEG:
                deg = d[a]
            elif op == MUL:
                deg = d[a] + d[b]
            i = len(self.nodes)
            self.nodes.append(key); d.append(deg); self._memo[key] = i
        return Expr(self, i)

    def constant(self, v: int) -> Expr:
        if isinstance(v, Expr):
            return v
        if not isinstance(v, (int, np.integer)):
            raise TypeError(f"constants are integers, got {type(v).__name__}")
        return self._node(CONST, imm=self.field.to_monty(int(v) % self.field.P))

    def main(self): return _Main(self, self.width)
    def preprocessed(self): return _Preprocessed(self, self.preprocessed_width)

    def periodic_values(self):
        return [self._node(PERIODIC, k) for k in range(self.num_periodic)]

    def public_values(self):
        return [self._node(PUBLIC, k) for k in range(self.num_public)]

    def is_first_row(self): return self._node(IS_FIRST_ROW)
    def is_last_row(self): return self._node(IS_LAST_ROW)
    def is_transition(self): return self._node(IS_TRANSITION)

    def assert_zero(self, x):
        x = self._e(x)
        if x.g is not self:
            raise ValueError("expression built by another builder")
        self.constraints.append(x.i)

    def node_array(self) -> np.ndarray:
        return np.array(self.nodes, dtype=np.uint32).reshape(-1, 4)


def _is_pow2(n: int) -> bool:
    return n > 0 and n & (n - 1) == 0


def periodic_column_error(periodic_columns, trace_length: int):
    """check_periodic_column_lengths (uni-stark/src/verifier.rs:25-50): None, or why a column cannot be evaluated over a trace
    of `trace_length` rows (a period that is not a power of two, or one longer than the trace)."""
    for k, col in enumerate(periodic_columns):
        p = len(col)
        if not _is_pow2(p):
            return f"periodic column {k}: period {p} is not a power of two"
        if p > trace_length:
            return f"periodic column {k}: period {p} exceeds the trace length {trace_length}"
    return None


class SymbolicAir:
    """An AIR given by `eval_fn(builder)`, in the surface uni_stark.prove and verifier.verify read.

    preprocessed_trace              (height, width) host (numpy uint32) or device matrix of Montgomery words: BaseAir::preprocessed_trace
    preprocessed_next_row_columns   the preprocessed columns read on the next row (default: all, air/src/air.rs:138-140); empty means
                                    the proof opens the preprocessed trace at zeta only
    periodic_columns                list of columns of canonical values, each of a power-of-two length (its period)"""

    def __init__(self, field: Field, width: int, eval_fn: Callable, num_public_values: int = 0,
                 main_next_row_columns: Optional[Sequence[int]] = None, max_constraint_degree: Optional[int] = None, gpu=None,
                 preprocessed_trace=None, preprocessed_next_row_columns: Optional[Sequence[int]] = None,
                 periodic_columns: Optional[Sequence[Sequence[int]]] = None):
        self.field, self.gpu = field, gpu
        self._pre_trace = preprocessed_trace
        pre_width = int(preprocessed_trace.shape[1]) if preprocessed_trace is not None else 0
        self._periodic = [[int(v) % field.P for v in col] for col in (periodic_columns or [])]
        for k, col in enumerate(self._periodic):
            if not _is_pow2(len(col)):
                raise ValueError(f"periodic column {k}: period {len(col)} is not a power of two")
        b = SymbolicAirBuilder(field, width, num_public_values, pre_width, len(self._periodic))
        eval_fn(b)
        self.builder = b
        self.nodes = b.node_array()
        self.constraints = np.array(b.constraints, dtype=np.uint32)
        # BaseAir::main_next_row_columns defaults to every column; it decides whether the proof carries the next-row opening
        self._next_cols = list(range(b.width)) if main_next_row_columns is None else [int(c) for c in main_next_row_columns]
        if not self._next_cols and any(n[0] == MAIN_NEXT for n in b.nodes):
            raise ValueError("the constraints read the next row but main_next_row_columns() is empty")
        self._pre_next_cols = (list(range(pre_width)) if preprocessed_next_row_columns is None
                               else [int(c) for c in preprocessed_next_row_columns])
        if not self._pre_next_cols and any(n[0] == PREPROCESSED_NEXT for n in b.nodes):
            raise ValueError("the constraints read the preprocessed next row but preprocessed_next_row_columns() is empty")
        self._degree_hint = max_constraint_degree
        self._program = None
        self._check_program = None
        self._periodic_tables = {}

    # ---- BaseAir / the degree the quotient is split by
    def width(self) -> int: return self.builder.width
    def num_public_values(self) -> int: return self.builder.num_public
    def main_next_row_columns(self): return list(self._next_cols)
    def preprocessed_width(self) -> int: return self.builder.preprocessed_width
    def preprocessed_trace(self): return self._pre_trace
    def preprocessed_next_row_columns(self): return list(self._pre_next_cols)
    def num_periodic_columns(self) -> int: return len(self._periodic)
    def periodic_columns(self): return [list(c) for c in self._periodic]

    def _has_layout(self) -> bool:
        return self.preprocessed_width() > 0 or self.num_periodic_columns() > 0

    def constraint_degrees(self):
        return [self.builder.degrees[c] for c in self.builder.constraints]

    def max_constraint_degree(self) -> int:
        """The hint if given (uni-stark/src/symbolic.rs), otherwise the largest degree_multiple of a constraint."""
        if self._degree_hint is not None:
            return int(self._degree_hint)
        return max(self.constraint_degrees(), default=0)

    # ---- prover: the quotient on the device
    def _need_gpu(self, what):
        if self.gpu is None:
            raise _lib.P3GpuError(f"{what} needs a GPU context (no CPU fallback)")

    def _to_device(self, t):
        """Host tensor `t` on the context's CUDA device (unchanged for a stand-in device without an integer `device`)."""
        if isinstance(getattr(self.gpu, "device", None), int):
            return t.to(f"cuda:{self.gpu.device}")
        return t

    def program(self):
        self._need_gpu("quotient evaluation")
        if self._program is None:
            if self._has_layout():
                layout = (self.width(), self.num_public_values(), self.preprocessed_width(), self.num_periodic_columns())
                self._program = self.gpu.air_program_create_layout(self.field.id, self.nodes, self.constraints, layout)
            else:
                self._program = self.gpu.air_program_create(self.field.id, self.nodes, self.constraints, self.width(), self.num_public_values())
        return self._program

    def check_program(self):
        """The AIR's constraints compiled for the debug check (p3gpu_air_check_program_create): no constraint limit, up to 65,535
        slots, so every hand-written AIR's DAG compiles too."""
        self._need_gpu("the constraint check")
        if self._check_program is None:
            layout = (self.width(), self.num_public_values(), self.preprocessed_width(), self.num_periodic_columns())
            self._check_program = self.gpu.air_check_program_create(self.field.id, self.nodes, self.constraints, layout)
        return self._check_program

    def constraint_label(self, k: int) -> Optional[str]:
        return self.builder.labels.get(int(k))

    def periodic_table(self, log_degree: int, log_quotient_size: int):
        """build_periodic_lde_table_two_adic (fri/src/periodic.rs:43-160) on the device: every column padded to the largest period
        p_max by repetition, coset-LDE'd onto p_max * 2^q rows (q = log_quotient_size - log_degree, the quotient domain's blowup) over
        the shift GENERATOR^(|K| / (p_max 2^q)), natural order: natural index i of the quotient domain reads row i mod (p_max 2^q).
        (p_max * 2^q, n_periodic) device matrix, built once per (trace height, quotient size); None without periodic columns."""
        if not self._periodic:
            return None
        key = (int(log_degree), int(log_quotient_size))
        if key not in self._periodic_tables:
            import torch
            f, n = self.field, 1 << log_degree
            err = periodic_column_error(self._periodic, n)
            if err:
                raise ValueError(err)
            p_max = max(len(c) for c in self._periodic)
            q = log_quotient_size - log_degree
            padded = np.array([[c[i % len(c)] for c in self._periodic] for i in range(p_max)], dtype=np.uint64)
            m = self._to_device(torch.from_numpy(f.to_monty_array(padded).astype(np.uint32).view(np.int32)))
            shift = f.pow(f.generator, n // p_max)                     # GENERATOR^(|K| / (p_max 2^q)), |K| = n 2^q
            self._periodic_tables[key] = self.gpu.coset_lde_batch(f.id, m, q, shift, bitrev_rows=False)
        return self._periodic_tables[key]

    def quotient_values(self, trace_lde_dev, log_degree: int, alpha, public_values=(), preprocessed_on_quotient_domain=None):
        """uni-stark/src/prover.rs:462-827: `trace_lde_dev` holds the trace on the quotient domain GENERATOR * K, |K| = its height, in
        bit-reversed row order (the committed LDE or its prefix).  Returns (|K|, 4) in natural order.  `public_values`: canonical.
        `preprocessed_on_quotient_domain`: the preprocessed trace the same way (required iff the AIR has preprocessed columns)."""
        if len(public_values) != self.num_public_values():
            raise ValueError(f"{len(public_values)} public values given, the AIR has {self.num_public_values()}")
        if (preprocessed_on_quotient_domain is not None) != (self.preprocessed_width() > 0):
            raise ValueError(f"the AIR has {self.preprocessed_width()} preprocessed columns: the preprocessed trace on the quotient domain "
                             f"is {'given' if preprocessed_on_quotient_domain is not None else 'missing'}")
        H = int(trace_lde_dev.shape[0])
        log_q = H.bit_length() - 1
        pv = [self.field.to_monty(int(v) % self.field.P) for v in public_values]
        if not self._has_layout():
            return self.gpu.air_quotient(self.program(), trace_lde_dev, log_q, log_degree, pv, alpha)
        table = self.periodic_table(log_degree, log_q)
        prog = self.program()
        return self.gpu.air_quotient_layout(prog, trace_lde_dev, preprocessed_on_quotient_domain, table, log_q, log_degree, pv, alpha)

    def sharded_quotient_values(self, grp, log_lde_height: int, log_degree: int, alpha, public_values=()):
        """The quotient values of `grp`'s row block after its sharded commit (distributed.PeerGroup.commit), over the LDE domain
        (log_num_quotient_chunks == log_blowup): (R, 4), R = 2^log_lde_height / world, in bit-reversed order: entry m is natural
        index bitrev(rank R + m).  Next-row columns are read from the row block of the one rank that holds them
        (distributed.next_row_rank).  `grp`: anything with the commit's `struct` (_lib.PeerGroupStruct) and `col_starts`.
        `public_values`: canonical.  No preprocessed columns."""
        if len(public_values) != self.num_public_values():
            raise ValueError(f"{len(public_values)} public values given, the AIR has {self.num_public_values()}")
        if self.preprocessed_width() > 0:
            raise ValueError(f"the AIR has {self.preprocessed_width()} preprocessed columns: no sharded quotient")
        log_lde_height, log_degree = int(log_lde_height), int(log_degree)
        pv = [self.field.to_monty(int(v) % self.field.P) for v in public_values]
        table = self.periodic_table(log_degree, log_lde_height)
        return self.gpu.air_quotient_sharded(self.program(), grp.struct, grp.col_starts, table, log_lde_height, log_degree, pv, alpha)

    # ---- verifier: the constraint folder on the same DAG
    def eval_folded_constraints(self, e, local, nxt, public_values, is_first_row, is_last_row, is_transition, alpha, *,
                                preprocessed_local=None, preprocessed_next=None, periodic_values=None):
        """VerifierConstraintFolder (uni-stark/src/folder.rs): acc = acc * alpha + c per constraint, on canonical EF4 values (`e`:
        verifier.Ext), every node evaluated once.  The preprocessed rows and periodic values at zeta are given when the AIR has
        them."""
        f = self.field
        vals = []
        for op, a, b, imm in self.builder.nodes:
            if op == CONST:
                v = e.base(f.from_monty(imm))
            elif op == MAIN_LOCAL:
                v = local[a]
            elif op == MAIN_NEXT:
                v = nxt[a]
            elif op == PUBLIC:
                v = e.base(int(public_values[a]))
            elif op == IS_FIRST_ROW:
                v = is_first_row
            elif op == IS_LAST_ROW:
                v = is_last_row
            elif op == IS_TRANSITION:
                v = is_transition
            elif op == PREPROCESSED_LOCAL:
                v = preprocessed_local[a]
            elif op == PREPROCESSED_NEXT:
                v = preprocessed_next[a]
            elif op == PERIODIC:
                v = periodic_values[a]
            elif op == ADD:
                v = e.add(vals[a], vals[b])
            elif op == SUB:
                v = e.sub(vals[a], vals[b])
            elif op == NEG:
                v = e.sub(e.ZERO, vals[a])
            else:
                v = e.mul(vals[a], vals[b])
            vals.append(v)
        acc = [0, 0, 0, 0]
        for c in self.builder.constraints:
            acc = e.add(e.mul(acc, alpha), vals[c])
        return acc


@dataclass(frozen=True)
class ConstraintFailure:
    """One violated constraint (air/src/check_constraints.rs ConstraintFailure): the row, the constraint's index in assertion order
    and the label of a named assertion."""
    row: int
    constraint: int
    label: Optional[str] = None

    def __str__(self):
        if self.label is None:
            return f"#{self.constraint}"
        return f"#{self.constraint} " + '"' + self.label.replace("\\", "\\\\").replace('"', '\\"') + '"'


@dataclass
class ConstraintReport:
    """check_all_constraints' result (ConstraintReport): the failures in row order, each row's in constraint order."""
    failures: List[ConstraintFailure]
    total_rows: int
    total_constraints_per_row: int

    def is_ok(self) -> bool:
        return not self.failures


class ConstraintViolation(ValueError):
    """check_constraints' failure: the first failing row and every constraint that failed on it."""

    def __init__(self, row: int, failures: List[ConstraintFailure]):
        self.row, self.failures = int(row), list(failures)
        super().__init__(f"constraints not satisfied on row {self.row}: failed constraints = [{', '.join(map(str, self.failures))}]")


def _device_matrix(air, m, what):
    """`m` (host numpy or device matrix of Montgomery words) as a contiguous int32 tensor on the AIR's device."""
    import torch
    if not isinstance(m, torch.Tensor):
        m = torch.from_numpy(np.ascontiguousarray(m, dtype=np.uint32).view(np.int32))
    if m.dim() != 2:
        raise ValueError(f"{what}: a matrix, got shape {tuple(m.shape)}")
    return air._to_device(m.to(torch.int32).contiguous())


def _check_inputs(air, trace, public_values):
    """What both passes read: the trace, the preprocessed trace (height checked as the reference asserts), the periodic table
    (each column repeated to the largest period) and the public values (Montgomery)."""
    air._need_gpu("the constraint check")
    if int(trace.dim()) != 2 or int(trace.shape[1]) != air.width():
        raise ValueError(f"trace of shape {tuple(trace.shape)}: the AIR has {air.width()} columns")
    height = int(trace.shape[0])
    if height < 1:
        raise ValueError("the trace has no rows")
    if len(public_values) != air.num_public_values():
        raise ValueError(f"{len(public_values)} public values given, the AIR has {air.num_public_values()}")
    pre = None
    if air.preprocessed_width() > 0:
        pre = _device_matrix(air, air.preprocessed_trace(), "preprocessed trace")
        if int(pre.shape[0]) != height:
            raise ValueError(f"the constraint check needs the preprocessed trace height ({int(pre.shape[0])}) to match the trace "
                             f"height ({height})")
    per = None
    cols = air.periodic_columns()
    if cols:
        p_max = max(len(c) for c in cols)
        padded = np.array([[c[i % len(c)] for c in cols] for i in range(p_max)], dtype=np.uint64)
        per = _device_matrix(air, air.field.to_monty_array(padded).astype(np.uint32), "periodic table")
    pv = [air.field.to_monty(int(v) % air.field.P) for v in public_values]
    return height, pre, per, pv


def _failures(air, trace, public_values, max_failures):
    """Both passes: the per-row counts on the device, then the failing constraints of the rows check_all_constraints would visit
    with this cap (the cap is tested before each row), selected on the device."""
    import torch
    height, pre, per, pv = _check_inputs(air, trace, public_values)
    prog, gpu = air.check_program(), air.gpu
    counts = gpu.air_check_counts(prog, trace, pre, per, pv).to(torch.int64)
    ends = torch.cumsum(counts, 0)
    before = ends - counts                                         # failures in the rows above each row
    keep = counts > 0
    if max_failures is not None:
        keep &= before < int(max_failures)
    rows = torch.nonzero(keep).flatten()
    n_rows = int(rows.numel())
    if n_rows == 0:
        return height, []
    offsets = (before[rows] - before[rows[0]]).contiguous()
    per_row = counts[rows]
    total = int(offsets[-1] + per_row[-1])
    failed = gpu.air_check_rows(prog, trace, pre, per, pv, rows.to(torch.int32).contiguous(), offsets, total)
    rows_h, per_row_h, failed_h = rows.cpu().numpy(), per_row.cpu().numpy(), failed.cpu().numpy()
    out, at = [], 0
    for r, c in zip(rows_h.tolist(), per_row_h.tolist()):
        out.extend(ConstraintFailure(r, k, air.constraint_label(k)) for k in failed_h[at:at + c].tolist())
        at += c
    return height, out


def check_all_constraints(air: "SymbolicAir", trace, public_values=(), max_failures: Optional[int] = None) -> ConstraintReport:
    """p3_air::check_all_constraints (air/src/check_constraints.rs:528-627) on the device: every constraint on every row of `trace`
    (a device int32 matrix of Montgomery words, any height >= 1, as for `prove`).  `public_values`: canonical integers.  With
    `max_failures`, rows stop being visited once that many failures are collected; the cap is tested between rows, so the last
    row's failures may overshoot it."""
    height, failures = _failures(air, trace, public_values, max_failures)
    return ConstraintReport(failures, height, len(air.constraints))


def check_constraints(air: "SymbolicAir", trace, public_values=()) -> None:
    """p3_air::check_constraints (air/src/check_constraints.rs:429-505) on the device: raises ConstraintViolation naming the first
    row with a failing constraint and every constraint that fails there."""
    _, failures = _failures(air, trace, public_values, 1)
    if failures:
        raise ConstraintViolation(failures[0].row, failures)


class KernelAir(SymbolicAir):
    """A SymbolicAir whose prover runs the AIR's own hand-written kernels instead of a constraint program: no public values, no
    preprocessed columns, no CPU fallback.  A subclass names the AIR in `air_name` and launches its quotient kernel in
    `_kernel_quotient`; one that can be proved row-sharded (distributed.prove_sharded) also launches its sharded quotient kernel in
    `_kernel_quotient_sharded`."""
    air_name = ""

    @classmethod
    def has_sharded_quotient(cls) -> bool:
        """Whether the AIR has a quotient kernel for one rank's row block of the row-sharded commit."""
        return cls._kernel_quotient_sharded is not KernelAir._kernel_quotient_sharded

    def sharded_quotient_values(self, grp, log_lde_height: int, log_degree: int, alpha, public_values=()):
        """The quotient values of `grp`'s row block after its sharded commit (distributed.PeerGroup.commit, log_blowup 1): (R, 4), R =
        2^log_lde_height / world, in bit-reversed order: entry m is natural index bitrev(rank R + m) of the quotient domain.  The AIR's
        own sharded kernel, never the constraint program; it takes no public values."""
        if len(public_values) != 0:
            raise ValueError(f"{len(public_values)} public values given, the {self.air_name} AIR has none")
        self._need_gpu("quotient evaluation")
        return self._kernel_quotient_sharded(grp, int(log_lde_height), int(log_degree), alpha)

    def _kernel_quotient_sharded(self, grp, log_lde_height: int, log_degree: int, alpha):
        raise NotImplementedError(f"the {self.air_name} AIR has no sharded quotient kernel")

    def quotient_values(self, trace_lde_dev, log_degree: int, alpha, public_values=(), preprocessed_on_quotient_domain=None):
        """uni-stark/src/prover.rs:462-827 on the AIR's hand-written kernel: `trace_lde_dev` holds the trace on the quotient domain in
        bit-reversed row order (the committed LDE or its prefix, as `_kernel_quotient` says).  Returns (|K|, 4) in natural order."""
        if len(public_values) != 0:
            raise ValueError(f"{len(public_values)} public values given, the {self.air_name} AIR has none")
        if preprocessed_on_quotient_domain is not None:
            raise ValueError(f"the {self.air_name} AIR has no preprocessed columns")
        self._need_gpu("quotient evaluation")
        return self._kernel_quotient(trace_lde_dev, log_degree, alpha)

    def _kernel_quotient(self, trace_lde_dev, log_degree: int, alpha):
        raise NotImplementedError
