"""Prove a trace whose LDE does not fit on one GPU beside it: the LDE is kept as the trace's coefficients plus one coset at a time.

Memory rows [k N, (k+1) N) of the committed bit-reversed LDE (N = trace height) are the evaluations on the coset
GENERATOR * w^bitrev(k) * H in bit-reversed order, w a generator of the 2^log_blowup-th roots of unity.  Each is one coset DFT of
the trace's coefficients (p3gpu_lde_coset_block_dev), it holds complete rows, so its leaf digests form a whole sub-tree of the trace
tree, and multiplying by w_N maps it to itself, so every point's next row lies in the same coset.  So the prover needs only the
coefficients (converted in the trace's own storage, p3gpu_lde_coefficients_dev) and one coset: about twice the trace, against
(1 + 2^log_blowup) times for the resident LDE.  Every step that reads the LDE recomputes the coset it needs.

CosetBlockedTrace is the one-GPU counterpart of distributed.ShardedTrace, with the cosets as its row blocks: it stands in for the
trace commit, the quotient values, the opening's two row steps and the trace's query openings, and `uni_stark.prove(config, air,
trace, shard=CosetBlockedTrace(gpu, config, air))` writes the proof `prove` writes, byte for byte.  A coset block is laid out as a row block of the
row-sharded commit with every column on one source (distributed.column_segments: column chunks, each a dense (N, chunk) matrix), which
is what the AIRs' sharded quotient kernels read; the Merkle leaves hash the chunks' rows in column order, which is hashing whole rows.
"""
from __future__ import annotations

import numpy as np
import torch

from .distributed import (PeerGroup, _split_error, block_openings, blocks_view, column_segments, natural_order,
                          segments_rowwise_dot)

MAX_BLOCKS = 16                     # the sharded quotient kernels' group holds at most 16 row blocks
MIN_BLOCK_ROWS = 1024               # ... of at least 1024 rows each, as the sharded commit's
MAX_CHUNK_COLUMNS = 128             # shard_chunk_bounds' column chunks are below 96 columns (64 by default)


def coset_blocked_error(config, air):
    """None, or why CosetBlockedTrace cannot prove `air` under `config`; decided on the host from the arguments alone.  It needs a
    StarkConfig, KeccakStarkConfig or Sha256StarkConfig, a quotient domain equal to the LDE domain (log_num_quotient_chunks ==
    log_blowup) and either an air.KernelAir with a sharded quotient kernel (the Poseidon2 AIR over KoalaBear, the Blake3, SHA-256 and
    Poseidon1 AIRs) or a constraint-program SymbolicAir without preprocessed columns."""
    from .uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig
    if not isinstance(config, (StarkConfig, KeccakStarkConfig, Sha256StarkConfig)):
        return f"CosetBlockedTrace: {type(config).__name__} is not a StarkConfig or KeccakStarkConfig, nor a Sha256StarkConfig"
    return _air_error(air, config.pcs.fri.log_blowup)


def _air_error(air, log_blowup: int):
    """coset_blocked_error's rules on the AIR and the blowup."""
    from .air import KernelAir, SymbolicAir
    from .field import KoalaBear
    from .poseidon2_air import VectorizedPoseidon2Air
    from .uni_stark import get_log_num_quotient_chunks
    head = "CosetBlockedTrace: "
    if not isinstance(air, SymbolicAir):
        return head + f"{type(air).__name__} is not an air.SymbolicAir"
    if isinstance(air, KernelAir):
        name = air.air_name or type(air).__name__
        if not air.has_sharded_quotient():
            return head + f"the {name} AIR has no sharded quotient kernel, which is what evaluates one coset block"
        if isinstance(air, VectorizedPoseidon2Air) and air.field.id != KoalaBear.id:
            return head + f"the Poseidon2 AIR over {air.field.name} has no sharded quotient kernel (KoalaBear only)"
    elif air.preprocessed_width() > 0:
        return head + f"the AIR has {air.preprocessed_width()} preprocessed columns, which coset blocks do not take"
    chunks = get_log_num_quotient_chunks(air)
    if chunks != log_blowup:
        return head + (f"log_num_quotient_chunks {chunks} (constraint degree {air.max_constraint_degree()}) differs from log_blowup "
                       f"{log_blowup}: coset blocks evaluate the quotient on the LDE domain only")
    if (1 << log_blowup) > MAX_BLOCKS:
        return head + f"log_blowup {log_blowup} gives {1 << log_blowup} cosets, more than the {MAX_BLOCKS} blocks the quotient kernels take"
    err = _split_error(air.width(), block_col_starts(air.width(), log_blowup))
    if err:
        return head + f"a trace of {air.width()} columns: {err}"
    return None


def block_col_starts(width: int, log_blowup: int):
    """The column offsets of a coset block's layout: every column on source 0 of 2^log_blowup."""
    return [0] + [int(width)] * (1 << log_blowup)


def coset_blocked_allowance_bytes(width: int, log_degree: int, log_blowup: int) -> int:
    """What CosetBlockedTrace's prove holds beside the coefficients and the one coset: the digest layers of every coset's sub-tree,
    the column chunk of coefficients the coset DFT reads, and the quotient and FRI vectors, each a small multiple of 16 bytes per LDE
    row (the quotient's bit-reversed and natural orders, its chunks' LDE and tree, the reduced openings, the folded layers); 64 bytes
    per LDE row per coset bounds them."""
    N, B = 1 << log_degree, 1 << log_blowup
    H = N * B
    digests = B * (2 * N - 1) * 32
    chunk = N * min(int(width), MAX_CHUNK_COLUMNS) * 4
    return digests + chunk + 64 * H * B


def coset_blocked_memory_bytes(air, log_degree: int, log_blowup: int) -> int:
    """The planned peak device memory of proving `air` on 2^log_degree rows with CosetBlockedTrace: the coefficients and one coset
    (twice the trace) plus `coset_blocked_allowance_bytes`.  `prove` holds the trace and its whole LDE instead, (1 + 2^log_blowup) times
    the trace, so a caller can choose between the two."""
    trace = (1 << log_degree) * int(air.width()) * 4
    return 2 * trace + coset_blocked_allowance_bytes(air.width(), log_degree, log_blowup)


class _CosetBlockGroup:
    """What an AIR's sharded quotient kernel reads of a row-sharded commit (distributed.PeerGroup): the group struct naming the row
    blocks, the column offsets and the block height.  Here the one resident coset stands for block `rank` of `world`; its next rows
    lie in the same block (distributed.next_row_rank with world = 2^log_blowup), so the view names it for every rank."""
    p2air_quotient = PeerGroup.p2air_quotient

    def __init__(self, gpu, world: int, rank: int, block, col_starts, rows: int):
        self.gpu, self.world, self.rank, self.rows_per_rank = gpu, world, rank, rows
        self.col_starts = col_starts
        self.struct = blocks_view(world, rank, [block] * world)


class CosetBlockedTrace:
    """The trace's prover data and its opener with the LDE held as coefficients plus one coset (see the module docstring).  Pass it
    as `uni_stark.prove(config, air, trace, shard=CosetBlockedTrace(gpu, config, air))`, or call `prove_coset_blocked`.  The trace given to prove is consumed: its storage holds the coefficients.  At most one coset is resident; the last one
    computed stays until another is needed, so consecutive steps over the same coset compute it once."""

    def __init__(self, gpu, config, air):
        """`gpu`: the config's GPU context.  Raises ValueError, before any device call, when coset_blocked_error refuses `config` or
        `air`."""
        err = coset_blocked_error(config, air)
        if err:
            raise ValueError(err)
        self.gpu, self.width = gpu, int(air.width())
        self.resident = None                           # the coset the block buffer holds

    # ---- the commit
    def commit(self, pcs, trace):
        """The trace's coefficients in place, then per coset: compute it, hash its rows into its sub-tree; the levels above the
        sub-tree roots from merkle_from_digests.  Returns (cap, prover data = self); the cap equals pcs.commit's."""
        from .dft import _log2_strict
        if int(trace.shape[0]) < MIN_BLOCK_ROWS:
            raise ValueError(f"CosetBlockedTrace: a trace of {int(trace.shape[0])} rows: the sharded quotient kernels take coset blocks of "
                             f"at least {MIN_BLOCK_ROWS} rows")
        gpu, f, mmcs = self.gpu, pcs.dft.field, pcs.mmcs
        self.field, self.hash_kind = f, mmcs.hash_kind
        m = gpu._dev(trace)
        N, W = int(m.shape[0]), self.width
        assert int(m.shape[1]) == W, f"a trace of {int(m.shape[1])} columns, the AIR has {W}"
        self.log_degree, self.log_blowup = _log2_strict(N), pcs.fri.log_blowup
        self.log_height = self.log_degree + self.log_blowup
        B = 1 << self.log_blowup
        self.rows, self.blocks = N, B
        self.shape, self.device = (N * B, W), m.device
        self.shift = f.div(f.generator, pcs.natural_domain_for_degree(N)[0])          # TwoAdicFriPcs.commit's coset shift
        self.col_starts = block_col_starts(W, self.log_blowup)
        bounds = column_segments(B, self.col_starts, N)
        self.block = torch.empty(N * W, dtype=torch.int32, device=m.device)
        self.segments = [(c0, c1, self.block[off:off + N * (c1 - c0)].view(N, c1 - c0)) for c0, c1, off in bounds]
        wmax = max(c1 - c0 for c0, c1, _ in bounds)
        # a coset DFT reads one column chunk of the coefficients, copied dense (none with one chunk: the coefficients are that chunk)
        self.piece = torch.empty(N * wmax, dtype=torch.int32, device=m.device) if len(bounds) > 1 else None
        for p in mmcs.perms:
            p.upload(gpu)
        self.coeffs = gpu.lde_coefficients(f.id, m)
        self.resident = None
        self.sub_layers = []
        for k in range(B):
            self._compute(k)
            self.sub_layers.append(gpu.merkle_commit(f.id, self.hash_kind, [blk for _, _, blk in self.segments]))
        roots = torch.stack([layers[-1][0] for layers in self.sub_layers])            # (B, 8): level log2(B) of the trace tree
        top = gpu.merkle_from_digests(f.id, self.hash_kind, roots) if B > 1 else [roots]
        self.top_layers = [t.cpu().numpy().view(np.uint32) for t in top]
        cap_height = min(mmcs.cap_height, self.log_height)
        if cap_height <= self.log_blowup:
            cap = self.top_layers[self.log_blowup - cap_height][: 1 << cap_height]
        else:                                          # the cap lies inside the sub-trees: each coset's slice of it, in order
            lvl = cap_height - self.log_blowup
            cap = np.concatenate([layers[len(layers) - 1 - lvl][: 1 << lvl].cpu().numpy().view(np.uint32) for layers in self.sub_layers])
        self.path_len = self.log_height - cap_height
        return np.ascontiguousarray(cap), self

    def _compute(self, k: int):
        """Make coset k the resident block: its coset DFT column chunk by column chunk, each straight into its segment."""
        if self.resident == k:
            return
        gpu, f, N = self.gpu, self.field, self.rows
        for c0, c1, seg in self.segments:
            if self.piece is None:
                src = self.coeffs
            else:
                src = self.piece[:N * (c1 - c0)].view(N, c1 - c0)
                src.copy_(self.coeffs[:, c0:c1])
            gpu.lde_coset_block(f.id, src, self.log_blowup, self.shift, k, out=seg)
        self.resident = k

    def _order(self, cosets):
        """`cosets` with the resident one first, so that it is not computed twice."""
        return sorted(cosets, key=lambda k: k != self.resident)

    # ---- the quotient
    def quotient_values(self, air, quotient_domain, alpha, public_values=()):
        """The AIR's quotient values in natural order over the quotient domain, which must be the LDE domain: per coset, the AIR's
        sharded quotient kernel on it as block k of a 2^log_blowup-block view, the slices put back in natural order by one gather."""
        assert quotient_domain[1] == self.log_height, "coset blocks evaluate the quotient on the LDE domain: log_num_quotient_chunks == log_blowup"
        N = self.rows
        q_bitrev = torch.empty((N * self.blocks, 4), dtype=torch.int32, device=self.device)
        for k in self._order(range(self.blocks)):
            self._compute(k)
            grp = _CosetBlockGroup(self.gpu, self.blocks, k, self.block, self.col_starts, N)
            q_bitrev[k * N:(k + 1) * N] = air.sharded_quotient_values(grp, self.log_height, self.log_degree, alpha, public_values)
        return natural_order(q_bitrev, self.log_height)

    # ---- the opening's row steps (fri._row_steps)
    def get_matrices(self, _data):
        return [self]

    def low_coset_dot(self, h, weights, scale):
        """columnwise_dot over the first h rows, which are coset 0's: per column segment, scaled."""
        assert h <= self.rows, "the low coset is memory block 0"
        gpu, f = self.gpu, self.field
        self._compute(0)
        ys = torch.empty((self.width, 4), dtype=torch.int32, device=self.device)
        for c0, c1, seg in self.segments:
            ys[c0:c1] = gpu.columnwise_dot(f.id, seg[:h], weights, scale)
        return ys

    def reduce_rows(self, acc, alpha, terms, coeff_and_yred):
        """The trace's reduced openings per coset: rowwise_dot per column segment times alpha^(first column), then open_reduce of
        every term into the coset's rows of `acc`."""
        gpu, f, N = self.gpu, self.field, self.rows
        coeffs = [(inv_denoms, *coeff_and_yred(offset, ys)) for inv_denoms, offset, ys in terms]
        for k in self._order(range(self.blocks)):
            self._compute(k)
            r = segments_rowwise_dot(gpu, f, self.segments, N, alpha)
            rows = slice(k * N, (k + 1) * N)
            for inv_denoms, coeff, yred in coeffs:
                gpu.open_reduce(f.id, acc[rows], r, inv_denoms[rows], coeff, yred)

    # ---- the query openings (prove_fri)
    def get_max_height(self, _data):
        return self.shape[0]

    def open_multi_batch(self, indices, _data):
        """Mmcs::open_multi_batch: per coset that holds a queried row (coset idx // N, local row idx % N), compute it and gather its
        queries' rows; the paths from the resident digest layers (the coset's sub-tree, then the levels above the sub-tree roots)."""
        N, W, plen = self.rows, self.width, self.path_len
        idx = np.asarray(indices, dtype=np.int64)
        n = int(idx.size)
        owner, local = idx // N, idx % N
        table = torch.zeros((n, W + plen * 8), dtype=torch.int32, device=self.device)
        for k in self._order(np.unique(owner).tolist()):
            self._compute(k)
            mine = np.nonzero(owner == k)[0]
            table[torch.from_numpy(mine).to(table.device)] = block_openings(self.gpu, self.segments, N, self.sub_layers[k],
                                                                            self.top_layers, k, local[mine], W, plen)
        ans = table.cpu().numpy().view(np.uint32)
        return [np.ascontiguousarray(ans[:, :W])], np.ascontiguousarray(ans[:, W:]).reshape(n, plen, 8)


def prove_coset_blocked(config, air, trace, public_values=()):
    """uni_stark.prove through CosetBlockedTrace on the config's GPU; coset_blocked_error's refusals raise ValueError naming the reason,
    before any device call.  Returns the Proof `prove` writes for the same trace, byte for byte.  `trace` (device, CUDA int32) is
    consumed: its storage holds the coefficients afterwards."""
    from .uni_stark import prove
    err = coset_blocked_error(config, air)
    if err:
        raise ValueError(err)
    return prove(config, air, trace, public_values, shard=CosetBlockedTrace(config.pcs.dft.gpu, config, air))
