"""Host arithmetic of the row-sharded prove that decides which rank owns what (no GPU call): the owner of a query's row, the
natural index of every entry of a rank's bit-reversed quotient slice, and the column-segment table the sharded quotient kernel
reads a chunk-major row block through."""
import numpy as np
import pytest

from plonky3_b200 import _lib
from plonky3_b200.distributed import column_segments, column_starts, query_owner, quotient_slice_natural_indices


def _bitrev(i, bits):
    return int(format(i, f"0{bits}b")[::-1], 2) if bits else 0


@pytest.mark.parametrize("log_h,world", [(11, 1), (11, 2), (12, 4), (21, 8)])
def test_query_owner(log_h, world):
    R = (1 << log_h) // world
    for idx in [0, 1, R - 1, R % (1 << log_h), (1 << log_h) - 1, (1 << log_h) // 3, 12345 % (1 << log_h)]:
        g, m = query_owner(idx, R)
        assert 0 <= g < world and 0 <= m < R and g * R + m == idx


@pytest.mark.parametrize("log_h,world", [(3, 1), (5, 2), (6, 4), (11, 8)])
def test_quotient_slice_natural_indices(log_h, world):
    H = 1 << log_h
    R = H // world
    nat = np.concatenate([quotient_slice_natural_indices(g, R, log_h) for g in range(world)])
    assert sorted(nat.tolist()) == list(range(H))                       # the slices together are a permutation of the domain
    assert [int(x) for x in nat] == [_bitrev(m, log_h) for m in range(H)]


def _check_segments(world, starts, rows):
    segs = column_segments(world, starts, rows)
    assert segs[0][0] == 0 and segs[-1][1] == starts[-1]
    assert all(a[1] == b[0] for a, b in zip(segs, segs[1:]))         # the segments tile the row in column order
    for c0, c1, off in segs:
        assert c0 < c1 and c0 % 4 == 0 and c1 % 4 == 0
        if world == 1:
            assert off == 0 and (c0, c1) == (0, starts[-1])
        else:
            g = max(q for q in range(world) if starts[q] <= c0)
            assert c1 <= starts[g + 1], "a segment never crosses a rank's column block"
            assert off == rows * c0                                    # chunk-major: the chunk's matrix starts at rows * c0
    return segs


@pytest.mark.parametrize("chunk", ["8", "16", "64", "100", "1312"])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_column_segments(world, chunk, monkeypatch):
    monkeypatch.setenv("P3GPU_SHARD_CHUNK", chunk)
    for width in (1312, 164, 328, 40):
        starts = column_starts(width, world, align=8)
        segs = _check_segments(world, starts, 1024)
        if world > 1:
            L = _lib.load()
            import ctypes as C
            n_chunks = 0
            for g in range(world):
                buf = (C.c_size_t * 400)()
                n = L.p3gpu_shard_chunk_bounds(starts[g + 1] - starts[g], buf, 400)
                n_chunks += sum(1 for i in range(n - 1) if buf[i + 1] > buf[i])
            assert len(segs) == n_chunks                               # one segment per exchanged chunk
    _check_segments(world, [0] + [4 * (k + 1) for k in range(world - 1)] + [4 * world + 1300], 2048)   # blocks of 4 columns


@pytest.mark.parametrize("world,starts", [(2, [0, 650, 1312]), (2, [0, 2, 1312]), (4, [0, 328, 656, 985, 1312]), (1, [0, 1310])])
def test_column_segments_reject_misaligned_layouts(world, starts):
    """A segment bound that is not a multiple of 4 columns would let a 16-byte load read across two chunks."""
    with pytest.raises(_lib.P3GpuError, match="multiple of 4"):
        column_segments(world, starts, 1024)


def test_column_segments_reject_bad_blocks():
    with pytest.raises(_lib.P3GpuError):
        column_segments(2, [0, 800, 640], 1024)                        # unordered
    with pytest.raises(_lib.P3GpuError):
        column_segments(2, [8, 640, 1312], 1024)                       # does not start at 0
