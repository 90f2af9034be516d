"""Multi-GPU commit of one trace across the ranks of a torch.distributed group (one process per GPU, NCCL over NVLink).

SURVEY.md section 8(e): the NTT/LDE shards by COLUMN (every column is an independent polynomial, dft/src/traits.rs:22-24),
the Merkle tree shards by ROW RANGE (a leaf digest is a sequential sponge over the whole row, merkle_tree.rs:309-317, and
rows [k*H/G, (k+1)*H/G) of the bit-reversed LDE form a complete sub-tree).  Two modes:

  commit_column_blocks   BASELINE's "independent NTT+Merkle per shard": every rank commits its own column block;
                         ONE all-gather of the G roots.  Each root equals the reference's commitment to that column block
                         alone (G commitments, not the reference's single-trace commitment).
  commit_bit_exact       the reference's single commitment: column-sharded LDE -> ONE all-to-all that re-shards column
                         blocks into row blocks -> local leaf hashing + sub-tree -> ONE all-gather of sub-tree roots ->
                         the top log2(G) levels are compressed redundantly on every rank.  Bit-identical to
                         TwoAdicFriPcs::commit on the whole trace.  With G = 2^cap_height (8 GPUs, cap_height 3 as in
                         examples/src/proofs.rs:150) the gathered sub-tree roots ARE the Merkle cap.

The compute backend is injected (`backend.lde`, `backend.commit_rows`, `backend.tree_from_digests`), so the sharding and
collective logic is testable with gloo on CPU; `GpuBackend` binds it to libp3gpu.
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist


def column_starts(width: int, world: int, align: int = 1):
    """The world + 1 offsets of the `column_block` split."""
    return [column_block(width, world, r, align)[0] for r in range(world)] + [width]


def column_block(width: int, world: int, rank: int, align: int = 1):
    """Contiguous column block of `rank` in units of `align` columns: the first (width/align) % world ranks get one extra
    unit, the last rank also takes the width % align remainder.  align = 8 keeps every 32-byte segment the LDE's last pass
    stores into a row block sector-aligned (DESIGN.md section 5)."""
    units, rem = divmod(width, align)
    base, extra = divmod(units, world)
    start = (rank * base + min(rank, extra)) * align
    stop = start + (base + (1 if rank < extra else 0)) * align
    if rank == world - 1:
        stop += rem
    return start, stop


class GpuBackend:
    """libp3gpu-backed compute (device-resident CUDA int32 tensors)."""

    def __init__(self, gpu, field, hash_kind, log_blowup):
        self.gpu, self.field, self.hash_kind, self.log_blowup = gpu, field, hash_kind, log_blowup

    def lde(self, evals):                       # (h, w_local) -> (h << log_blowup, w_local), bit-reversed rows
        return self.gpu.coset_lde_batch(self.field.id, evals, self.log_blowup, self.field.generator, bitrev_rows=True)

    def commit_rows(self, mats):                # list of same-height matrices (one per source rank) -> digest layers
        return self.gpu.merkle_commit(self.field.id, self.hash_kind, mats)

    def tree_from_digests(self, digests):       # (n, 8) -> layers above
        return self.gpu.merkle_from_digests(self.field.id, self.hash_kind, digests)


def _all_gather(t: torch.Tensor, group=None) -> List[torch.Tensor]:
    world = dist.get_world_size(group)
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t.contiguous(), group=group)
    return out


def _all_to_all(recv: List[torch.Tensor], send: List[torch.Tensor], group=None):
    """NCCL: one all_to_all.  Backends without it (gloo, used by the CPU tests): pairwise isend/irecv."""
    if dist.get_backend(group) == "nccl":
        dist.all_to_all(recv, send, group=group)
        return
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    recv[rank].copy_(send[rank])
    reqs = []
    for k in range(world):
        if k != rank:
            reqs.append(dist.isend(send[k], dst=dist.get_global_rank(group, k) if group is not None else k, group=group))
            reqs.append(dist.irecv(recv[k], src=dist.get_global_rank(group, k) if group is not None else k, group=group))
    for r in reqs:
        r.wait()


def commit_column_blocks(backend, evals_local: torch.Tensor, group=None):
    """Independent LDE + Merkle per column block; one all-gather of roots.  Returns (roots (G, 8), lde_local, layers_local)."""
    lde = backend.lde(evals_local)
    layers = backend.commit_rows([lde])
    roots = torch.stack(_all_gather(layers[-1][0].contiguous(), group))
    return roots, lde, layers


def commit_bit_exact(backend, evals_local: torch.Tensor, widths: List[int], cap_height: int, group=None):
    """Bit-exact single commitment of the column-sharded trace.  `widths[g]` = columns held by rank g.
    Returns (cap (2^cap_height-ish, 8), lde_rows: list of per-source-rank row-block matrices, local sub-tree layers)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    assert world & (world - 1) == 0, "row sharding needs a power-of-two number of ranks"
    lde = backend.lde(evals_local)                                   # (H, w_rank), bit-reversed rows
    H = lde.shape[0]
    assert H % world == 0
    rows = H // world
    # all-to-all: rank g sends rows [k*rows, (k+1)*rows) of its column block to rank k
    send = [lde[k * rows:(k + 1) * rows].contiguous() for k in range(world)]
    recv = [torch.empty((rows, widths[g]), dtype=lde.dtype, device=lde.device) for g in range(world)]
    _all_to_all(recv, send, group)
    # the G received pieces, in rank order, are exactly the column blocks of my rows: hashing their row-wise concatenation
    # is hashing the full-width row (MerkleTree::new with several matrices of one height, merkle_tree.rs:312-316)
    layers = backend.commit_rows(recv)
    sub_root = layers[-1][0].contiguous()
    roots = torch.stack(_all_gather(sub_root, group))                # (G, 8): level log2(G) of the global tree
    top = backend.tree_from_digests(roots)                           # [roots, ..., global root]
    log_g = world.bit_length() - 1
    if cap_height <= log_g:
        cap = top[log_g - cap_height][: 1 << cap_height]
    else:                                                            # cap below the sub-tree roots: gather my slice of it
        h_local = cap_height - log_g
        eff = min(h_local, len(layers) - 1)
        piece = layers[len(layers) - 1 - eff][: 1 << eff].contiguous()
        cap = torch.cat(_all_gather(piece, group))
    return cap, recv, layers


# ------------------------------------------------------------------------------------------------------------------
# Peer-memory mode: no collective library on the data path (csrc/peer.cu, include/p3gpu.h "multi-GPU")
# ------------------------------------------------------------------------------------------------------------------
import ctypes as C

import numpy as np

from . import _lib
from . import extension as X
from ._lib import check


class RawBuffer:
    """Device memory from p3gpu_malloc (plain cudaMalloc: exportable through CUDA IPC, unlike a slice of torch's caching
    allocator).  `tensor(shape)` views it as a CUDA int32 tensor without copying."""

    def __init__(self, gpu, nbytes: int):
        self.gpu, self.nbytes = gpu, int(nbytes)
        p = C.c_void_p()
        check(gpu.L.p3gpu_malloc(gpu.h, self.nbytes, C.byref(p)))
        self.ptr = p.value

    def tensor(self, shape):
        n = int(np.prod(shape))
        assert n * 4 <= self.nbytes
        holder = type("_CudaArray", (), {})()
        holder.__cuda_array_interface__ = {"shape": tuple(int(x) for x in shape), "typestr": "<i4", "data": (self.ptr, False), "version": 3}
        holder._keepalive = self
        return torch.as_tensor(holder, device=f"cuda:{self.gpu.device}")

    def free(self):
        if self.ptr:
            check(self.gpu.L.p3gpu_free(self.gpu.h, C.c_void_p(self.ptr)))
            self.ptr = None


class PeerGroup:
    """One rank's view of the group: its control block and row block plus every peer's, mapped through CUDA IPC.

    rows_per_rank x w_total is the shape of the row block each rank hashes (rows_per_rank = LDE height / world).
    Bootstrap = one all_gather_object of two 64-byte IPC handles per rank over torch.distributed (host side, once);
    afterwards no collective library call is made on the data path."""

    def __init__(self, gpu, rows_per_rank: int, w_total: int, group=None, timeout_s: float = 20.0, _sim=None):
        self.gpu, self.rows_per_rank, self.w_total = gpu, int(rows_per_rank), int(w_total)
        self.epoch = C.c_uint32(0)
        self._imported = []
        self.group, self._simulated = group, _sim is not None
        self.xchg, self.xchg_ptrs, self._xchg_imported = None, None, []
        if _sim is not None:                       # single-process simulation (tests): all blocks live on this device
            self.world, self.rank, self.ctrl, self.rows, peers = _sim
        else:
            self.world = dist.get_world_size(group) if dist.is_initialized() else 1
            self.rank = dist.get_rank(group) if dist.is_initialized() else 0
            self.ctrl = RawBuffer(gpu, _lib.PEER_CTRL_BYTES)
            self.rows = RawBuffer(gpu, self.rows_per_rank * self.w_total * 4)
            check(gpu.L.p3gpu_ctx_use_own_stream(gpu.h))
            check(gpu.L.p3gpu_memset_dev(gpu.h, C.c_void_p(self.ctrl.ptr), 0, _lib.PEER_CTRL_BYTES))
            gpu.sync()
            peers = [(self.ctrl.ptr, self.rows.ptr)] * self.world
            if self.world > 1:
                hc, hr = (C.c_uint8 * 64)(), (C.c_uint8 * 64)()
                check(gpu.L.p3gpu_ipc_export(gpu.h, C.c_void_p(self.ctrl.ptr), hc))
                check(gpu.L.p3gpu_ipc_export(gpu.h, C.c_void_p(self.rows.ptr), hr))
                handles = [None] * self.world
                dist.all_gather_object(handles, (bytes(hc), bytes(hr)), group=group)
                peers = []
                for q, (bc, br) in enumerate(handles):
                    if q == self.rank:
                        peers.append((self.ctrl.ptr, self.rows.ptr))
                        continue
                    pc, pr = C.c_void_p(), C.c_void_p()
                    check(gpu.L.p3gpu_ipc_import(gpu.h, (C.c_uint8 * 64).from_buffer_copy(bc), C.byref(pc)))
                    check(gpu.L.p3gpu_ipc_import(gpu.h, (C.c_uint8 * 64).from_buffer_copy(br), C.byref(pr)))
                    self._imported += [pc.value, pr.value]
                    peers.append((pc.value, pr.value))
                dist.barrier(group=group)          # every control block is zeroed and mapped before the first device barrier
        self.struct = _lib.PeerGroupStruct()
        self.struct.world, self.struct.rank, self.struct.timeout_s = self.world, self.rank, timeout_s
        for q, (pc, pr) in enumerate(peers):
            self.struct.ctrl[q], self.struct.rows[q] = pc, pr

    @classmethod
    def simulate(cls, gpus, rows_per_rank: int, w_total: int, timeout_s: float = 10.0):
        """`len(gpus)` ranks inside ONE process on ONE device (one libp3gpu context = one stream per rank): lets a 1-GPU box
        exercise the sharded kernels, the barrier and the all-gather bit for bit.  Ranks must be driven from separate host
        threads, each under its own torch.cuda.stream (the barrier kernel spins until every rank has arrived: two ranks on
        one stream would dead-lock until the watchdog fires)."""
        world = len(gpus)
        ctrl = [RawBuffer(g, _lib.PEER_CTRL_BYTES) for g in gpus]
        rows = [RawBuffer(g, rows_per_rank * w_total * 4) for g in gpus]
        for g, c in zip(gpus, ctrl):
            check(g.L.p3gpu_ctx_use_own_stream(g.h))
            check(g.L.p3gpu_memset_dev(g.h, C.c_void_p(c.ptr), 0, _lib.PEER_CTRL_BYTES))
            g.sync()
        peers = [(c.ptr, r.ptr) for c, r in zip(ctrl, rows)]
        return [cls(g, rows_per_rank, w_total, timeout_s=timeout_s, _sim=(world, q, ctrl[q], rows[q], peers)) for q, g in enumerate(gpus)]

    def rows_tensor(self):
        return self.rows.tensor((self.rows_per_rank, self.w_total))

    def barrier(self):
        self.gpu._use_torch_stream()
        self.epoch.value += 1
        check(self.gpu.L.p3gpu_peer_barrier_dev(self.gpu.h, C.byref(self.struct), self.epoch.value))

    def lde_sharded(self, field, evals_local, added_bits: int, shift: int, col_off: int):
        """p3gpu_coset_lde_batch_sharded_dev on torch's current stream (complete on all ranks after the next barrier)."""
        m = self.gpu._dev(evals_local); self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_coset_lde_batch_sharded_dev(self.gpu.h, field.id, C.byref(self.struct), m.data_ptr(), m.shape[0], m.shape[1],
                                                          added_bits, shift, self.w_total, col_off))

    def commit(self, field, hash_kind: int, evals_local, col_starts, log_blowup: int, cap_height: int, phases: bool = False):
        """p3gpu_commit_sharded_dev.  `col_starts`: world + 1 column offsets (rank g holds [col_starts[g], col_starts[g+1]));
        an int is taken as my own offset of an even `column_block` split, for callers that do not know the others' blocks.
        Returns (cap (n, 8) uint32 array — identical on every rank, my sub-tree's digest layers as CUDA tensors,
        [lde_ms, barrier_ms, hash_ms, cap_exchange_ms] or None).  With world > 1 my row block is left chunk-major
        (`row_block_dense` reassembles it)."""
        gpu = self.gpu
        m = gpu._dev(evals_local)                                    # (h, w_local); w_local may be 0 (more ranks than column units)
        h, w_local = int(m.shape[0]), int(m.shape[1])
        assert (h << log_blowup) == self.rows_per_rank * self.world
        if isinstance(col_starts, int):
            raise TypeError("PeerGroup.commit needs the world + 1 column offsets of all ranks (column_starts(...))")
        starts = [int(x) for x in col_starts]
        assert len(starts) == self.world + 1 and starts[-1] == self.w_total and starts[self.rank + 1] - starts[self.rank] == w_local
        self.col_starts = starts
        cs = (C.c_size_t * (self.world + 1))(*starts)
        gpu._use_torch_stream()
        tot = gpu.merkle_total_digests(self.rows_per_rank)
        layers = gpu._empty((tot, 8))
        lens = (C.c_size_t * 65)(); nl = C.c_size_t()
        cap = np.zeros((max(1 << cap_height, self.world), 8), dtype=np.uint32); cap_len = C.c_size_t()
        ph = (C.c_float * 4)() if phases else None
        check(gpu.L.p3gpu_commit_sharded_dev(gpu.h, field.id, hash_kind, C.byref(self.struct), C.byref(self.epoch), m.data_ptr(), h, cs,
                                             log_blowup, cap_height, layers.data_ptr(), lens, C.byref(nl),
                                             cap.ctypes.data, C.byref(cap_len), ph))
        out, off = [], 0
        for k in range(nl.value):
            out.append(layers[off:off + lens[k]]); off += lens[k]
        return cap[: cap_len.value].copy(), out, ([float(x) for x in ph] if phases else None)

    def chunk_bounds(self, w_local: int):
        b = (C.c_size_t * (w_local // 8 + 3))()
        n = self.gpu.L.p3gpu_shard_chunk_bounds(w_local, b, len(b))
        return [int(b[i]) for i in range(n)]

    def row_block_dense(self, col_starts=None):
        """My row block as a dense (rows_per_rank, w_total) tensor (a copy), whatever layout the last commit left it in."""
        starts = col_starts if col_starts is not None else self.col_starts
        R = self.rows_per_rank
        if self.world == 1:
            return self.rows_tensor().clone()
        flat = self.rows_tensor().reshape(-1)
        out = torch.empty((R, self.w_total), dtype=flat.dtype, device=flat.device)
        for g in range(self.world):
            cb = self.chunk_bounds(starts[g + 1] - starts[g])
            for a, b in zip(cb[:-1], cb[1:]):
                if b > a:
                    c0 = starts[g] + a
                    out[:, c0:c0 + (b - a)] = flat[R * c0: R * (c0 + b - a)].reshape(R, b - a)
        return out

    def column_segments(self, col_starts=None):
        """[(first column, end column, element offset)] of my row block as the last commit left it (p3gpu_shard_col_segments)."""
        return column_segments(self.world, col_starts if col_starts is not None else self.col_starts, self.rows_per_rank)

    def ensure_exchange(self, nbytes: int):
        """Collective: every rank's exchange buffer holds at least `nbytes`, mapped on every rank through CUDA IPC.  A smaller
        buffer from an earlier call is closed and replaced; every rank must call this with the same size."""
        if self.xchg is not None and self.xchg.nbytes >= nbytes:
            return
        if self._simulated:
            raise NotImplementedError("exchange buffers need one process per rank")
        self._close_exchange()
        self.xchg = RawBuffer(self.gpu, nbytes)
        ptrs = [self.xchg.ptr] * self.world
        if self.world > 1:
            h = (C.c_uint8 * 64)()
            check(self.gpu.L.p3gpu_ipc_export(self.gpu.h, C.c_void_p(self.xchg.ptr), h))
            handles = [None] * self.world
            dist.all_gather_object(handles, bytes(h), group=self.group)
            for q, b in enumerate(handles):
                if q != self.rank:
                    p = C.c_void_p()
                    check(self.gpu.L.p3gpu_ipc_import(self.gpu.h, (C.c_uint8 * 64).from_buffer_copy(b), C.byref(p)))
                    self._xchg_imported.append(p.value)
                    ptrs[q] = p.value
        self.xchg_ptrs = (C.c_void_p * 16)(*ptrs)

    def exchange(self, src):
        """p3gpu_peer_exchange_dev: all-gather of `src` (contiguous CUDA int32) over the exchange buffers.  Returns a
        (world, src.numel()) view of MY exchange buffer, valid until the next exchange."""
        s = self.gpu._dev(src)
        words = int(s.numel())
        assert self.xchg is not None and self.world * words * 4 <= self.xchg.nbytes, "exchange buffer too small (ensure_exchange)"
        self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_peer_exchange_dev(self.gpu.h, C.byref(self.struct), C.byref(self.epoch), self.xchg_ptrs, s.data_ptr(), words))
        return self.xchg.tensor((self.world, words))

    def p2air_quotient(self, field, vector_len: int, log_lde_height: int, log_trace_height: int, alpha):
        """p3gpu_p2air_quotient_sharded_dev on my row block: (rows_per_rank, 4) quotient values, bit-reversed slice `rank`."""
        gpu = self.gpu
        gpu._use_torch_stream()
        cs = (C.c_size_t * (self.world + 1))(*self.col_starts)
        q = gpu._empty((self.rows_per_rank, 4))
        check(gpu.L.p3gpu_p2air_quotient_sharded_dev(gpu.h, field.id, vector_len, C.byref(self.struct), cs, log_lde_height, log_trace_height,
                                                     gpu._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    def _close_exchange(self):
        if self.xchg is None:
            return
        if self.world > 1 and not self._simulated:
            dist.barrier(group=self.group)         # no peer still copies into the buffer being freed
        for p in self._xchg_imported:
            self.gpu.L.p3gpu_ipc_close(self.gpu.h, C.c_void_p(p))
        self._xchg_imported = []
        self.xchg.free()
        self.xchg, self.xchg_ptrs = None, None

    def close(self):
        self._close_exchange()
        for p in self._imported:
            self.gpu.L.p3gpu_ipc_close(self.gpu.h, C.c_void_p(p))
        self._imported = []


def column_segments(world: int, col_starts, rows: int):
    """p3gpu_shard_col_segments: the (first column, end column, element offset) segments of a row block of `rows` rows after
    p3gpu_commit_sharded_dev with these column blocks.  Raises P3GpuError for a layout whose segment bounds are not multiples
    of 4 columns."""
    L = _lib.load()
    starts = (C.c_size_t * (world + 1))(*[int(x) for x in col_starts])
    cap = 3 * (int(col_starts[-1]) // 4 + world + 2)
    buf = (C.c_size_t * cap)(); n = C.c_size_t()
    check(L.p3gpu_shard_col_segments(world, starts, rows, buf, cap // 3, C.byref(n)))
    return [(int(buf[3 * k]), int(buf[3 * k + 1]), int(buf[3 * k + 2])) for k in range(n.value)]


def chunk_major_block(rows_dense, world: int, col_starts):
    """Rows of the bit-reversed LDE laid out as p3gpu_commit_sharded_dev leaves a row block (`column_segments`): a flat CUDA int32
    tensor, the inverse of PeerGroup.row_block_dense.  Lets one GPU build the block any rank of a `world`-rank commit would hash."""
    R = int(rows_dense.shape[0])
    out = torch.empty(R * int(rows_dense.shape[1]), dtype=rows_dense.dtype, device=rows_dense.device)
    for c0, c1, off in column_segments(world, col_starts, R):
        out[off:off + R * (c1 - c0)] = rows_dense[:, c0:c1].reshape(-1)
    return out


def block_view(world: int, rank: int, block):
    """A _lib.PeerGroupStruct that names only my row block `block` (a CUDA tensor in the layout of `chunk_major_block`), for the
    sharded quotient entry points, which read nothing but grp->rows[rank].  The other ranks' row and control pointers are set to the
    same block to pass the group's null checks; nothing that exchanges, synchronises or hashes may be given this view."""
    st = _lib.PeerGroupStruct()
    st.world, st.rank, st.timeout_s = world, rank, 1.0
    for q in range(world):
        st.ctrl[q] = st.rows[q] = block.data_ptr()
    return st


def blocks_view(world: int, rank: int, blocks):
    """A _lib.PeerGroupStruct that names every rank's row block, `blocks[q]` (CUDA tensors in the layout of `chunk_major_block`,
    all on this device), as rank `rank` of a `world`-rank commit sees them: for the sharded quotient entry points, which read the own
    block and, for a constraint program that reads the next row, the block of `next_row_rank`.  The control pointers are set to the
    blocks to pass the group's null checks; nothing that exchanges, synchronises or hashes may be given this view."""
    st = _lib.PeerGroupStruct()
    st.world, st.rank, st.timeout_s = world, rank, 1.0
    for q in range(world):
        st.ctrl[q] = st.rows[q] = blocks[q].data_ptr()
    return st


def next_row_rank(rank: int, world: int, q: int) -> int:
    """The one rank holding the next rows of every point of `rank`'s row block (air_program.cuh air_shard_next_rank): point i =
    bitrev(M) of memory row M reads natural index i + 2^q, and the owner of a row is the low log2(world) bits of its natural index,
    bitrev(rank) for all of rank's points, so the owner is bitrev((bitrev(rank) + 2^q) mod world).  `rank` itself when world <= 2^q."""
    log_g = world.bit_length() - 1
    assert world == 1 << log_g and 0 <= rank < world, "world is a power of two, rank below it"
    if (1 << q) >= world:
        return rank
    return int(_bitrev((int(_bitrev(rank, log_g)) + (1 << q)) % world, log_g))


def query_owner(index: int, rows_per_rank: int):
    """(rank, local row) holding row `index` of the bit-reversed LDE after the row-sharded commit."""
    return index // rows_per_rank, index % rows_per_rank


def quotient_slice_natural_indices(rank: int, rows_per_rank: int, log_height: int):
    """Natural quotient-domain index of every entry of rank `rank`'s sharded quotient slice: bitrev(rank * R + m)."""
    m = np.arange(rank * rows_per_rank, (rank + 1) * rows_per_rank, dtype=np.int64)
    return _bitrev(m, log_height)


def natural_order(q_bitrev, log_height: int):
    """The quotient values of the whole domain in natural order from their 2^log_height bit-reversed entries (the row blocks' slices
    in block order): one gather."""
    H = 1 << log_height
    return q_bitrev[_bitrev(torch.arange(H, device=q_bitrev.device, dtype=torch.int64), log_height)].contiguous()


def segments_rowwise_dot(gpu, f, segments, rows: int, alpha):
    """Mred(x) = sum_c alpha^c M[x][c] for every row of a row block held as column segments [(c0, c1, (rows, c1 - c0) tensor)]:
    rowwise_dot per segment times alpha^c0, summed.  Returns (rows, 4)."""
    r = torch.zeros((rows, 4), dtype=torch.int32, device=segments[0][2].device)
    for c0, c1, block in segments:
        gpu.ef_axpy(f.id, r, gpu.rowwise_dot(f.id, block, alpha), X.ef_pow(f, alpha, c0))
    return r


def block_openings(gpu, segments, rows: int, sub_layers, top_layers, block: int, local, width: int, path_len: int):
    """Mmcs::open_multi_batch answers for queries at rows `local` of row block `block` of a tree whose row blocks are sub-trees: a
    (k, width + path_len * 8) tensor of each query's row and path.  The row is gathered from the block's column segments [(c0, c1,
    (rows, c1 - c0) tensor)], the path's levels inside the sub-tree come from the block's digest layers `sub_layers`, the levels above
    it from `top_layers` (host arrays: level l holds the 2^(log2(blocks) - l) digests over the sub-tree roots)."""
    li = np.ascontiguousarray(local, dtype=np.uint32)
    k = int(li.size)
    sub_len = min(rows.bit_length() - 1, path_len)
    out = torch.zeros((k, width + path_len * 8), dtype=torch.int32, device=segments[0][2].device)
    gpu._use_torch_stream()
    for c0, c1, blk in segments:
        piece = gpu._empty((k, c1 - c0))
        check(gpu.L.p3gpu_gather_rows_dev(gpu.h, blk.data_ptr(), rows, c1 - c0, li.ctypes.data, k, 0, piece.data_ptr()))
        out[:, c0:c1] = piece
    if sub_len:
        lens = (C.c_size_t * len(sub_layers))(*[int(l.shape[0]) for l in sub_layers])
        paths = gpu._empty((k, sub_len, 8))
        check(gpu.L.p3gpu_merkle_paths_dev(gpu.h, sub_layers[0].data_ptr(), lens, len(sub_layers), sub_len, li.ctypes.data, k, 0,
                                           paths.data_ptr()))
        out[:, width:width + sub_len * 8] = paths.reshape(k, -1)
    for lvl in range(path_len - sub_len):              # levels above the sub-tree roots: the same siblings for all the block's queries
        sib = np.ascontiguousarray(top_layers[lvl][(block >> lvl) ^ 1], dtype=np.uint32)
        out[:, width + (sub_len + lvl) * 8: width + (sub_len + lvl + 1) * 8] = torch.from_numpy(sib.view(np.int32)).to(out.device)
    return out


def _bitrev(x, bits: int):
    """Bit reversal of `bits`-bit indices: numpy int64 arrays or CUDA int64 tensors."""
    r = x * 0
    for b in range(bits):
        r = r | (((x >> b) & 1) << (bits - 1 - b))
    return r


class ShardedTrace:
    """The trace's prover data and its opener when the trace's columns are split over the ranks of a PeerGroup: rank g holds
    columns [col_starts[g], col_starts[g+1]), and after the sharded commit LDE rows [g R, (g+1) R), R = LDE height / world, with
    its sub-tree.  `uni_stark.prove(config, air, block, shard=ShardedTrace(grp, col_starts))` proves with it any air.KernelAir that
    has a sharded quotient kernel (the Poseidon2 AIR over KoalaBear, the Blake3, SHA-256 and Poseidon1 AIRs) and any
    constraint-program SymbolicAir without preprocessed columns (its next rows come from one peer's row block), under any
    configuration: the commit, the exchanges and the openings carry 8-word digests, which is what the Poseidon2, the Keccak and the
    SHA-256 MMCS write ([F; 8], [u64; 4] and [u8; 32]).

    It carries out the steps that read the trace's rows.  Ranks exchange data over peer memory only where a value depends on rows
    they do not own, and after every exchange all ranks hold identical bytes, so their transcripts stay identical:
      commit, quotient_values           prove's two branches: the sharded commit; the sharded quotient kernel on the own rows;
      low_coset_dot, reduce_rows        the two per-matrix steps of TwoAdicFriPcs.open_values_and_fri_inputs (fri._row_steps);
      get_max_height, open_multi_batch  the trace's query openings in prove_fri."""

    def __init__(self, grp: "PeerGroup", col_starts):
        self.grp, self.col_starts = grp, [int(x) for x in col_starts]
        self.width = self.col_starts[-1]

    def commit(self, pcs, trace_block):
        """PeerGroup.commit of my column block.  Returns (cap, prover data = self); the cap is identical on every rank."""
        from .dft import _log2_strict
        grp, mmcs, gpu = self.grp, pcs.mmcs, self.grp.gpu
        self.field, self.gpu = pcs.dft.field, gpu
        self.log_degree = _log2_strict(int(trace_block.shape[0]))
        self.log_height = self.log_degree + pcs.fri.log_blowup
        H, W, world = 1 << self.log_height, self.width, grp.world
        self.shape, self.device = (H, W), f"cuda:{gpu.device}"
        for p in mmcs.perms:
            p.upload(gpu)
        grp.ensure_exchange(4 * max(H * 4, world * W * 4, world * pcs.fri.num_queries * (W + 8 * self.log_height)))
        cap, self.sub_layers, _ = grp.commit(self.field, mmcs.hash_kind, trace_block, self.col_starts, pcs.fri.log_blowup, mmcs.cap_height)
        flat, R = grp.rows_tensor().reshape(-1), grp.rows_per_rank
        self.segments = [(c0, c1, flat[off:off + R * (c1 - c0)].reshape(R, c1 - c0)) for c0, c1, off in grp.column_segments()]
        log_g = world.bit_length() - 1
        self.top_layers = []
        if mmcs.cap_height < log_g:                  # the tree over the sub-tree roots, as the commit left it in the control block
            user = grp.ctrl.tensor((_lib.PEER_CTRL_BYTES // 4,))[_lib.PEER_CTRL_USER // 4:].cpu().numpy().view(np.uint32)
            off = world * 8
            for lvl in range(log_g):
                n = world >> lvl
                self.top_layers.append(user[off:off + n * 8].reshape(n, 8).copy()); off += n * 8
        self.path_len = self.log_height - min(mmcs.cap_height, self.log_height)
        return cap, self

    def quotient_values(self, air, quotient_domain, alpha, public_values=()):
        """The AIR's quotient values in natural order over the quotient domain, which must be the LDE domain: the AIR's sharded
        kernel on my rows in place, the bit-reversed slices all-gathered and put back in natural order by one gather."""
        assert quotient_domain[1] == self.log_height, "the sharded quotient covers the LDE domain: log_num_quotient_chunks == log_blowup"
        H = self.shape[0]
        q_slice = air.sharded_quotient_values(self.grp, self.log_height, self.log_degree, alpha, public_values)
        return natural_order(self.grp.exchange(q_slice).reshape(H, 4), self.log_height)

    def get_matrices(self, _data):
        return [self]

    def low_coset_dot(self, h, weights, scale):
        """columnwise_dot over the first h rows: each rank's unscaled partial over the rows it owns, all-gathered, summed with
        ef_axpy and scaled.  Field addition is exact, so the result equals the single-GPU value bit for bit."""
        grp, gpu, f = self.grp, self.gpu, self.field
        W, R = self.width, grp.rows_per_rank
        row0 = grp.rank * R
        partial = torch.zeros((W, 4), dtype=torch.int32, device=self.device)
        used = min(R, h - row0)
        if used > 0:
            for c0, c1, block in self.segments:
                partial[c0:c1] = gpu.columnwise_dot(f.id, block[:used], weights[row0:row0 + used])
        parts = grp.exchange(partial.reshape(-1)).reshape(grp.world, W, 4)
        acc = torch.zeros((W, 4), dtype=torch.int32, device=self.device)
        for q in range(grp.world):
            gpu.ef_axpy(f.id, acc, parts[q], X.ef_one(f))
        ys = torch.zeros((W, 4), dtype=torch.int32, device=self.device)
        gpu.ef_axpy(f.id, ys, acc, scale)
        return ys

    def reduce_rows(self, acc, alpha, terms, coeff_and_yred):
        """The trace's reduced openings over my rows: rowwise_dot per column segment times alpha^(first column), open_reduce of
        every term into my row slice of `acc`, then that slice all-gathered over the whole of `acc`."""
        grp, gpu, f = self.grp, self.gpu, self.field
        R = grp.rows_per_rank
        mine = slice(grp.rank * R, (grp.rank + 1) * R)
        r = segments_rowwise_dot(gpu, f, self.segments, R, alpha)
        for inv_denoms, offset, ys in terms:
            gpu.open_reduce(f.id, acc[mine], r, inv_denoms[mine], *coeff_and_yred(offset, ys))
        acc.copy_(grp.exchange(acc[mine]).reshape(acc.shape))

    def get_max_height(self, _data):
        return self.shape[0]

    def open_multi_batch(self, indices, _data):
        """Mmcs::open_multi_batch: every rank gathers the rows and authentication paths of the queries it owns (rank idx // R,
        local row idx % R), the tables are all-gathered over peer memory, and every rank takes each answer from its owner's slot.
        The path's levels inside a sub-tree come from the owner's sub-tree; the levels above it (cap_height < log2(world)) from
        the tree over the sub-tree roots that the commit left in the control block."""
        grp, gpu = self.grp, self.gpu
        R, W, rank = grp.rows_per_rank, grp.w_total, grp.rank
        idx = np.asarray(indices, dtype=np.int64)
        n, plen = int(idx.size), self.path_len
        owner, local = idx // R, idx % R
        mine = np.nonzero(owner == rank)[0]
        rec = W + plen * 8
        table = torch.zeros((n, rec), dtype=torch.int32, device=self.device)
        if mine.size:
            table[torch.from_numpy(mine).to(table.device)] = block_openings(gpu, self.segments, R, self.sub_layers, self.top_layers, rank,
                                                                             local[mine], W, plen)
        got = grp.exchange(table.reshape(-1)).reshape(grp.world, n, rec)
        ans = got[torch.from_numpy(owner).to(table.device), torch.arange(n, device=table.device)].cpu().numpy().view(np.uint32)
        return [np.ascontiguousarray(ans[:, :W])], np.ascontiguousarray(ans[:, W:]).reshape(n, plen, 8)


def _split_error(width: int, col_starts):
    """None, or why the sharded commit (p3gpu_commit_sharded_dev) and the sharded constraint-program quotient cannot take a trace of
    `width` columns split at `col_starts` (None: one rank).  The device's rules, decided on the host from the arguments alone:
      * ntt_coset_lde_sharded: every column block, its offset and the width are multiples of 4 columns;
      * its column-block LDE runs on the tiled pipeline (lde_tiled_impl), which takes at least 8 columns: the whole width at world 1
        (the single rank's fused LDE), every non-empty block otherwise;
      * air_shard_units: every segment of the chunk-major row block (shard_col_segments) starts on a multiple of 8 columns and ends on
        one or at the width, so no 8-column unit spans two segments."""
    starts = [0, width] if col_starts is None else [int(x) for x in col_starts]
    world = len(starts) - 1
    if world < 1 or world > 16 or world & (world - 1):
        return f"{world} ranks: a power of two up to 16"
    if starts[0] != 0 or starts[-1] != width or any(b < a for a, b in zip(starts, starts[1:])):
        return f"column blocks {starts} do not split the {width} columns in order"
    if width % 4:
        return "the sharded commit's LDE takes multiples of 4 columns"
    for g in range(world):
        a, b = starts[g], starts[g + 1]
        if a % 4 or b % 4:
            return f"rank {g}'s column block [{a}, {b}) does not start and end on a multiple of 4 columns, as the sharded commit's LDE needs"
        if 0 < b - a < 8:
            return (f"rank {g}'s column block [{a}, {b}) has {b - a} columns, fewer than the 8 the sharded commit's tiled LDE takes"
                    if world > 1 else f"fewer than the 8 columns the sharded commit's tiled LDE takes")
    try:
        segments = column_segments(world, starts, 1)
    except _lib.P3GpuError as e:
        return f"column blocks {starts}: {e}"
    for c0, c1, _ in segments:
        if c0 % 8 or (c1 % 8 and c1 != width):
            return (f"column blocks {starts} leave a row-block segment [{c0}, {c1}) that cuts an 8-column unit of the sharded quotient's "
                    "unit table")
    return None


def _symbolic_sharded_error(config, air, col_starts):
    """sharded_air_error for a constraint-program SymbolicAir: every decision from the arguments, before any device call, so every
    rank reaches the same one."""
    from .uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig, get_log_num_quotient_chunks
    head = f"prove_sharded: SymbolicAir is a constraint-program AIR of {air.width()} columns; "
    if air.preprocessed_width() > 0:
        return head + (f"it has {air.preprocessed_width()} preprocessed columns, which would need a sharded commit of the preprocessed "
                       "trace")
    err = _split_error(air.width(), col_starts)
    if err:
        return head + err
    if not isinstance(config, (StarkConfig, KeccakStarkConfig, Sha256StarkConfig)):
        return head + f"{type(config).__name__} is not a StarkConfig or KeccakStarkConfig, nor a Sha256StarkConfig"
    chunks, log_blowup = get_log_num_quotient_chunks(air), config.pcs.fri.log_blowup
    if chunks != log_blowup:
        return head + (f"log_num_quotient_chunks {chunks} (constraint degree {air.max_constraint_degree()}) differs from log_blowup "
                       f"{log_blowup}: the sharded quotient covers the LDE domain only")
    return None


def sharded_air_error(config, air, col_starts=None):
    """None, or why prove_sharded cannot prove `air` under `config` with the column blocks `col_starts` (None: not yet known; the
    rules that depend on them are checked at world 1): it needs a StarkConfig, KeccakStarkConfig or Sha256StarkConfig and either an
    air.KernelAir with a sharded quotient kernel whose constraints read the local row only (a row's next row lies on another rank),
    or a constraint-program SymbolicAir without preprocessed columns, whose quotient domain is the LDE domain and whose columns the
    sharded commit can take split at `col_starts`."""
    from .air import KernelAir, SymbolicAir
    from .field import KoalaBear
    from .poseidon2_air import VectorizedPoseidon2Air
    from .uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig
    if not isinstance(air, SymbolicAir):
        return f"prove_sharded: {type(air).__name__} is not an air.SymbolicAir"
    if not isinstance(air, KernelAir):
        return _symbolic_sharded_error(config, air, col_starts)
    name = air.air_name or type(air).__name__
    if air.main_next_row_columns():
        return f"prove_sharded: the {name} AIR reads the next row, which lies on another rank"
    if not air.has_sharded_quotient():
        return f"prove_sharded: the {name} AIR has no sharded quotient kernel"
    if isinstance(air, VectorizedPoseidon2Air) and air.field.id != KoalaBear.id:
        # its sharded quotient kernel reads 16-byte units of 4-column segments; BabyBear's 298-column permutations start mid-unit
        return f"prove_sharded: the Poseidon2 AIR over {air.field.name} has no sharded prove (KoalaBear only)"
    if not isinstance(config, (StarkConfig, KeccakStarkConfig, Sha256StarkConfig)):
        return f"prove_sharded: {type(config).__name__} is not a StarkConfig or KeccakStarkConfig, nor a Sha256StarkConfig"
    return None


def prove_sharded(config, air, grp: "PeerGroup", trace_block, col_starts, public_values=()):
    """uni_stark.prove with the trace sharded by column block over the ranks of `grp` (rank g holds columns [col_starts[g],
    col_starts[g+1]) of the 2^n-row trace), through ShardedTrace.  `config`: StarkConfig, KeccakStarkConfig or Sha256StarkConfig; `air`: the Poseidon2
    AIR over KoalaBear, the Blake3, SHA-256 or Poseidon1 AIR over either field, or a constraint-program SymbolicAir (next-row reads,
    public values and periodic columns included; sharded_air_error says why another is refused, before any device work).  Every rank
    returns the same Proof, byte for byte the one `uni_stark.prove` writes for the whole trace on one GPU; its timings_ms are each
    span's maximum over the ranks."""
    from .air import KernelAir
    from .uni_stark import get_log_num_quotient_chunks, prove
    err = sharded_air_error(config, air, col_starts)
    if err:
        raise ValueError(err)
    pcs = config.pcs
    assert grp.gpu is pcs.dft.gpu, "the PeerGroup and the config must share one GPU context"
    if isinstance(air, KernelAir):
        assert len(public_values) == 0, f"the {air.air_name} AIR has no public values"
    assert get_log_num_quotient_chunks(air) == pcs.fri.log_blowup, "quotient domain must equal the LDE domain (fast path of get_evaluations_on_domain)"
    proof = prove(config, air, trace_block, public_values, shard=ShardedTrace(grp, col_starts))
    if grp.world > 1 and dist.is_initialized():
        every = [None] * grp.world
        dist.all_gather_object(every, proof.timings_ms, group=grp.group)
        proof.timings_ms = {k: max(t[k] for t in every) for k in proof.timings_ms}
    return proof
