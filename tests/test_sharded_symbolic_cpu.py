"""The row-sharded prove of constraint-program SymbolicAirs without a GPU: the owner arithmetic of next rows, prove_sharded's guard,
and the sharded quotient's per-rank evaluation run on the host.

* `next_row_rank`: for every memory row M of the bit-reversed LDE, the rank holding M's next row, bitrev(bitrev(M) + 2^q), is
  next_row_rank(M // R): one rank per rank, a permutation, the rank itself iff world <= 2^q.
* The guard (`sharded_air_error` / `prove_sharded`) accepts and refuses from its arguments alone, before any device call.
* tests/cpp/air_shard_check.cpp runs air_program.cuh's air_row_quotient over every rank's chunk-major row block, addressed through
  the unit table and the owner helpers the kernel uses; every rank's slice must equal the oracle (tests/air_oracle.py) at the
  slice's natural indices, word for word."""
import os
import pathlib
import subprocess

import numpy as np
import pytest

import air_oracle as A
import sharded_symbolic_examples as S
from plonky3_b200.air import SymbolicAir
from plonky3_b200.distributed import (_bitrev, column_segments, column_starts, next_row_rank, prove_sharded,
                                      quotient_slice_natural_indices, sharded_air_error)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig

ROOT = pathlib.Path(__file__).resolve().parent.parent


class Untouchable:
    """A stand-in for the device, the peer group and the PCS: any use fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work before the refusal: .{name}")


class _Fri:
    def __init__(self, log_blowup):
        self.log_blowup = log_blowup


class _Pcs:
    """A PCS stand-in that answers only log_blowup."""

    def __init__(self, log_blowup):
        self.fri = _Fri(log_blowup)

    def __getattr__(self, name):
        raise AssertionError(f"device work before the refusal: .pcs.{name}")


# ---- next_row_rank ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_h", [11, 12, 13, 14])
def test_next_row_rank_holds_every_next_row(log_h):
    M = np.arange(1 << log_h, dtype=np.int64)
    for world in range(1, 17):
        if world & (world - 1):
            continue
        R = (1 << log_h) // world
        for q in (1, 2, 3):
            nxt = _bitrev((_bitrev(M, log_h) + (1 << q)) % (1 << log_h), log_h)
            owner = np.array([next_row_rank(g, world, q) for g in range(world)], dtype=np.int64)
            assert np.array_equal(nxt // R, owner[M // R]), (world, q)
            assert np.array_equal(owner == np.arange(world), np.full(world, world <= (1 << q))), (world, q)
            assert sorted(owner.tolist()) == list(range(world)), (world, q)


def test_next_row_rank_at_log_blowup_1():
    """World 2 reads no peer; worlds 4 to 16 read one peer each."""
    assert [next_row_rank(g, 2, 1) for g in range(2)] == [0, 1]
    for world in (4, 8, 16):
        assert all(next_row_rank(g, world, 1) != g for g in range(world))


# ---- the guard -------------------------------------------------------------------------------------------------------------
def _fib(b):
    m = b.main()
    b.when_transition().assert_eq(m.local[1], m.next[0])


CONFIGS = {"poseidon2": lambda lb: StarkConfig(_Pcs(lb), None), "keccak": lambda lb: KeccakStarkConfig(_Pcs(lb)),
           "sha256": lambda lb: Sha256StarkConfig(_Pcs(lb))}


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_the_64_column_air_is_accepted(config, world):
    air = S.wide_mul(KoalaBear)
    starts = column_starts(64, world, align=8)
    assert sharded_air_error(CONFIGS[config](1), air, starts) is None
    assert sharded_air_error(CONFIGS[config](2), S.wide_mul(BabyBear, degree=5), starts) is None


def test_public_values_and_periodic_columns_are_accepted():
    for world in (1, 2, 4):
        assert sharded_air_error(CONFIGS["poseidon2"](1), S.wide_fib(BabyBear), column_starts(32, world, align=8)) is None
        assert sharded_air_error(CONFIGS["keccak"](1), S.periodic(KoalaBear), column_starts(32, world, align=8)) is None
    assert sharded_air_error(CONFIGS["keccak"](1), S.periodic(KoalaBear)) is None          # column blocks not known yet: world 1


HEAD = "prove_sharded: SymbolicAir is a constraint-program AIR of {} columns; "


@pytest.mark.parametrize("case", ["preprocessed", "degree-5-at-blowup-1", "60-columns-world-8", "cut-unit", "width-2", "too-narrow"])
def test_refused_before_any_device_call(case):
    config = CONFIGS["poseidon2"](1)
    if case == "preprocessed":
        pre = np.zeros((8, 4), dtype=np.uint32)
        air = SymbolicAir(KoalaBear, 64, S.wide_mul_eval(), preprocessed_trace=pre)
        starts, message = column_starts(64, 2, align=8), HEAD.format(64) + "it has 4 preprocessed columns"
    elif case == "degree-5-at-blowup-1":
        air, starts = S.wide_mul(KoalaBear, degree=5), column_starts(64, 4, align=8)
        message = HEAD.format(64) + r"log_num_quotient_chunks 2 \(constraint degree 5\) differs from log_blowup 1"
    elif case == "60-columns-world-8":
        air, starts = SymbolicAir(KoalaBear, 60, S.wide_mul_eval(60)), column_starts(60, 8, align=8)
        assert starts[-2:] == [56, 60]
        message = HEAD.format(60) + r"rank 7's column block \[56, 60\) has 4 columns, fewer than the 8"
    elif case == "cut-unit":
        air, starts = S.wide_mul(KoalaBear), [0, 28, 64]
        message = HEAD.format(64) + r"column blocks \[0, 28, 64\] leave a row-block segment \[0, 28\) that cuts an 8-column unit"
    elif case == "width-2":
        air, starts = SymbolicAir(KoalaBear, 2, _fib), [0, 2]
        message = HEAD.format(2) + "the sharded commit's LDE takes multiples of 4 columns"
    else:
        air, starts = SymbolicAir(KoalaBear, 4, _fib), [0, 4]
        message = HEAD.format(4) + "fewer than the 8 columns the sharded commit's tiled LDE takes"
    with pytest.raises(ValueError, match=message):
        prove_sharded(config if case == "degree-5-at-blowup-1" else StarkConfig(Untouchable(), None), air, Untouchable(), Untouchable(),
                      starts)
    assert sharded_air_error(config, air, starts) is not None


def test_an_unknown_configuration_is_refused():
    with pytest.raises(ValueError, match="SymbolicAir is a constraint-program AIR of 64 columns; object is not a StarkConfig"):
        prove_sharded(object(), S.wide_mul(KoalaBear), Untouchable(), Untouchable(), [0, 64])


# ---- host execution of the per-rank quotient ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = tmp_path_factory.mktemp("air_shard") / "air_shard_check"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "air_shard_check.cpp"), "-o", str(exe)],
                   check=True)
    return exe


def _run(exe, f, air, lde, log_q, log_n, world, starts, pubs, alpha):
    R = (1 << log_q) // world
    segs = column_segments(world, starts, R)
    nodes = np.asarray(air.nodes, dtype=np.uint32).reshape(-1, 4)
    cons = np.asarray(air.constraints, dtype=np.uint32).ravel()
    job = [f.id, air.width(), air.num_public_values(), nodes.shape[0], cons.size, *nodes.ravel().tolist(), *cons.tolist(), log_q, log_n,
           world, len(segs), *[v for s in segs for v in s], *np.asarray(lde).ravel().tolist(), *pubs, *np.asarray(alpha).tolist()]
    out = subprocess.run([str(exe)], input=" ".join(map(str, job)), capture_output=True, text=True, check=True).stdout.split("\n")
    rc, misplaced = (int(v) for v in out[0].split())
    return rc, misplaced, [np.array(out[1 + g].split(), dtype=np.uint32).reshape(R, 4) for g in range(world)]


AIRS = {"mul64-deg3": (lambda f: S.wide_mul(f), 1), "mul64-deg5": (lambda f: S.wide_mul(f, degree=5), 2),
        "fib32-publics": (lambda f: S.wide_fib(f), 1)}


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("field", [BabyBear, KoalaBear], ids=["bb", "kb"])
@pytest.mark.parametrize("name", sorted(AIRS))
def test_every_rank_slice_matches_the_oracle(checker, name, field, world):
    make, q = AIRS[name]
    air = make(field)
    log_n = 4
    log_q = log_n + q
    rng = np.random.default_rng(world * 7 + q)
    lde = field.to_monty_array(rng.integers(0, field.P, (1 << log_q, air.width())).astype(np.uint64)).astype(np.uint32)
    pubs = [field.to_monty(int(v)) for v in rng.integers(0, field.P, air.num_public_values())]
    alpha = field.to_monty_array(rng.integers(0, field.P, 4).astype(np.uint64)).astype(np.uint32)
    starts = column_starts(air.width(), world, align=8)
    rc, misplaced, slices = _run(checker, field, air, lde, log_q, log_n, world, starts, pubs, alpha)
    assert rc == 0 and misplaced == 0
    exp = A.air_quotient(field.id, air.nodes, air.constraints, lde, log_q, log_n, pubs, alpha)
    R = (1 << log_q) // world
    for g in range(world):
        nat = quotient_slice_natural_indices(g, R, log_q)
        bad = np.flatnonzero((slices[g] != exp[nat]).any(axis=1))
        assert bad.size == 0, f"rank {g}: {bad.size} of {R} rows differ, first local row {bad[:1]}"
