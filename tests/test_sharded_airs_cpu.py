"""The row-sharded prove's AIR guard and its column-address arithmetic, without a GPU.

prove_sharded refuses, with a message naming the AIR and before any device call, an AIR that reads the next row (Keccak-f), a
constraint-program SymbolicAir, the Poseidon2 AIR over BabyBear and a configuration it does not know.  The sharded quotient kernels
read a chunk-major row block through a table of 8-column units (air_program.cuh AirShardRow): a Python model of that table, built
from the library's segment list, must put every column of every row where the chunk-major layout has it, and every 2- or 4-word
load of the kernels must stay inside one unit, for the Blake3, SHA-256 and Poseidon1 widths, where BabyBear's 298-column Poseidon1
permutations straddle chunk bounds."""
import numpy as np
import pytest

from plonky3_b200.air import SymbolicAir
from plonky3_b200.blake3_air import Blake3Air
from plonky3_b200.distributed import column_segments, column_starts, prove_sharded, sharded_air_error
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.keccak_air import KeccakAir
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air
from plonky3_b200.sha256_air import Sha256Air
from plonky3_b200.uni_stark import KeccakStarkConfig, StarkConfig


class Untouchable:
    """A stand-in for the device, the peer group and the PCS: any use fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work before the refusal: .{name}")


def _poseidon2(field, rounds_p):
    rng = np.random.default_rng(5)
    return VectorizedPoseidon2Air(field, RoundConstants(rng.integers(0, field.P, (4, 16)), rng.integers(0, field.P, rounds_p),
                                                        rng.integers(0, field.P, (4, 16))), None)


def _fib(b):
    m = b.main()
    b.when_transition().assert_eq(m.local[1], m.next[0])


@pytest.mark.parametrize("config", [StarkConfig(Untouchable(), None), KeccakStarkConfig(Untouchable())], ids=["poseidon2", "keccak"])
@pytest.mark.parametrize("air,message", [
    (KeccakAir(KoalaBear), "the Keccak AIR reads the next row"),
    (SymbolicAir(KoalaBear, 2, _fib), "SymbolicAir is a constraint-program AIR"),
    (_poseidon2(BabyBear, 13), f"the Poseidon2 AIR over {BabyBear.name} has no sharded prove"),
], ids=["keccak-f", "symbolic", "poseidon2-babybear"])
def test_refused_before_any_device_call(config, air, message):
    with pytest.raises(ValueError, match=message):
        prove_sharded(config, air, Untouchable(), Untouchable(), [0, air.width()])


def test_an_unknown_configuration_is_refused():
    with pytest.raises(ValueError, match="is not a StarkConfig or KeccakStarkConfig"):
        prove_sharded(object(), Blake3Air(KoalaBear), Untouchable(), Untouchable(), [0, 9168])


@pytest.mark.parametrize("config", [StarkConfig(Untouchable(), None), KeccakStarkConfig(Untouchable())], ids=["poseidon2", "keccak"])
@pytest.mark.parametrize("air", [Blake3Air(BabyBear), Sha256Air(KoalaBear), _poseidon2(KoalaBear, 20)], ids=["blake3", "sha256", "poseidon2"])
def test_the_sharded_airs_are_accepted(config, air):
    assert sharded_air_error(config, air) is None


# ---- the unit table --------------------------------------------------------------------------------------------------------
UNIT = 8


def _unit_table(world, starts, rows):
    """air_shard_units: per 8-column unit (base, stride) with column c of block row m at base + m * stride + c."""
    width = starts[-1]
    units = [None] * (-(-width // UNIT))
    for c0, c1, off in column_segments(world, starts, rows):
        assert c0 % UNIT == 0 and (c1 % UNIT == 0 or c1 == width), "a segment bound inside a unit"
        for u in range(c0 // UNIT, -(-c1 // UNIT)):
            units[u] = (off - c0, c1 - c0)
    assert all(e is not None for e in units)
    return units


def _chunk_major(dense, world, starts):
    """The row block as p3gpu_commit_sharded_dev leaves it (the layout distributed.chunk_major_block builds on the device)."""
    R = dense.shape[0]
    out = np.full(dense.size, -1, dtype=np.int64)
    for c0, c1, off in column_segments(world, starts, R):
        out[off:off + R * (c1 - c0)] = dense[:, c0:c1].ravel()
    return out


# the AIRs' widths: Blake3, SHA-256, Poseidon1 over KoalaBear (8 x 164) and over BabyBear (8 x 298)
WIDTHS = {"blake3": (9168, None), "sha256": (7728, None), "poseidon1-kb": (1312, 164), "poseidon1-bb": (2384, 298)}


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("air", sorted(WIDTHS))
def test_unit_table_addresses_every_column(air, world):
    width, perm = WIDTHS[air]
    rows = 16
    starts = column_starts(width, world, align=8)
    dense = np.arange(rows * width, dtype=np.int64).reshape(rows, width)
    flat = _chunk_major(dense, world, starts)
    units = _unit_table(world, starts, rows)
    base = np.array([units[c // UNIT][0] for c in range(width)], dtype=np.int64)
    stride = np.array([units[c // UNIT][1] for c in range(width)], dtype=np.int64)
    cols = np.arange(width, dtype=np.int64)
    for m in range(rows):
        assert np.array_equal(flat[base + m * stride + cols], dense[m])
    if perm is not None:
        # the Poseidon1 kernel's loads: 4 words at 4-aligned columns (KoalaBear), 2 words at even columns (BabyBear); each stays in
        # its unit, so its words are consecutive in memory, and starts as aligned as in the dense trace
        vec = 4 if perm % 4 == 0 else 2
        for v in range(width // perm):
            for c in range(v * perm, (v + 1) * perm, vec):
                assert c // UNIT == (c + vec - 1) // UNIT
                e0, e1 = units[c // UNIT]
                assert (e0 + c) % vec == 0 and (e1 * rows) % vec == 0 or world == 1
        if air == "poseidon1-bb" and world > 1:
            bounds = {c0 for c0, _, _ in column_segments(world, starts, rows)}
            assert any(v * perm < b < (v + 1) * perm for b in bounds for v in range(width // perm)), "no permutation straddles a chunk"
