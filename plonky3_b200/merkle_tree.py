"""MerkleTreeMmcs on the GPU: mirrors merkle-tree/src/mmcs/mod.rs:71 + mmcs/batch.rs:22-128 (Mmcs impl) and
merkle_tree.rs:33-217 (MerkleTree).  commit runs on the device; get_matrices/open_batch are host-side pointer chasing
over the stored digest layers, as in the reference."""
from __future__ import annotations

from dataclasses import dataclass, field as dc_field
from typing import List, Optional

import numpy as np

from . import _lib
from .field import Field
from .gpu import Gpu, default_gpu, _is_torch
from .poseidon2 import Poseidon2


def _log2_ceil(n: int) -> int:
    return max(n - 1, 0).bit_length()


@dataclass
class MerkleTree:
    """merkle_tree.rs:33-69: leaves (insertion order), every digest layer, arity schedule (always 2 here)."""
    leaves: list
    digest_layers: list          # layer 0 = leaf digests ... last = [root]; each (len, 8)
    arity_schedule: List[int] = dc_field(default_factory=list)

    def root(self):
        return _host(self.digest_layers[-1][0:1])[0]

    def cap(self, cap_height: int):
        """merkle_tree.rs:198-217."""
        n = len(self.digest_layers)
        if cap_height >= n:
            raise ValueError(f"cap_height {cap_height} exceeds tree depth {n}")
        layer = self.digest_layers[n - 1 - cap_height]
        return _host(layer[: min(1 << cap_height, layer.shape[0])])

    def num_layers(self):
        return len(self.digest_layers)


def _host(x):
    if _is_torch(x):
        return x.cpu().numpy().view(np.uint32)
    return np.array(x, dtype=np.uint32)


def _boundary_walk(indices, num_levels: int):
    """The frontier walk both directions of the pruned multiproof share (merkle-tree/src/pruning.rs:116-176, binary schedule):
    the sorted distinct leaf indices fold up level by level; a node whose sibling is not itself on the frontier needs that
    sibling from the proof.  Yields (level, slot) in wire order — level 0 first, ascending parent index inside a level — where
    `slot` is the position (in the caller's `indices`) of the smallest queried leaf under the node, whose full path holds the
    sibling at `level`."""
    first = {}
    for slot, i in enumerate(indices):
        first.setdefault(int(i), slot)
    nodes = sorted(first.items())                                     # (node index at this level, lead slot)
    for level in range(num_levels):
        parents, k = [], 0
        while k < len(nodes):
            idx, lead = nodes[k]
            if k + 1 < len(nodes) and nodes[k + 1][0] == (idx ^ 1):   # both children known: the verifier recomputes the parent
                k += 2
            else:
                yield level, lead
                k += 1
            parents.append((idx >> 1, lead))
        nodes = parents


def prune_paths(indices, paths) -> np.ndarray:
    """prune_paths (merkle-tree/src/pruning.rs:194-232): the minimal set of sibling digests of a batch of full paths.
    `paths`: (n, levels, 8), sibling digests bottom-up for `indices[q]`.  Returns (k, 8) in the reference's wire order."""
    paths = np.asarray(paths, dtype=np.uint32)
    out = [paths[slot, level] for level, slot in _boundary_walk(indices, paths.shape[1])]
    return np.array(out, dtype=np.uint32).reshape(len(out), 8)


def restore_paths(indices, pruned, num_levels: int) -> np.ndarray:
    """restore_paths (merkle-tree/src/pruning.rs:234-330): scatter the boundary digests back into the lead paths.  Positions
    the amortised verifier recomputes itself stay zero.  Raises ValueError when the digest count does not match the frontier."""
    pruned = np.asarray(pruned, dtype=np.uint32).reshape(-1, 8)
    full = np.zeros((len(indices), num_levels, 8), dtype=np.uint32)
    k = 0
    for level, slot in _boundary_walk(indices, num_levels):
        if k >= pruned.shape[0]:
            raise ValueError("pruned proof is shorter than its frontier")
        full[slot, level] = pruned[k]; k += 1
    if k != pruned.shape[0]:
        raise ValueError(f"pruned proof holds {pruned.shape[0]} digests, the frontier needs {k}")
    return full


class MerkleTreeError(Exception):
    """merkle-tree/src/mmcs/mod.rs MerkleTreeError (WrongBatchSize, WrongWidth, WrongHeight, IndexOutOfBounds, CapMismatch, ...)."""


def verify_multi_batch_with(hash_rows, compress_pairs, cap, dims, indices, opened_values, pruned):
    """verify_batch_pruned (merkle-tree/src/mmcs/mod.rs:430-): ONE amortised check of all queries of a batch.  Every distinct
    opened leaf is hashed once; the frontier folds up level by level — a sibling comes from the multiproof only where no queried
    leaf covers it, otherwise it was just computed; shorter matrices are injected where the level reaches their height
    (compress(node, hash(rows)), merkle_tree.rs:348-); every proof digest must be consumed and every surviving node must equal its
    cap entry.  `hash_rows((n, w) words) -> (n, 8)` and `compress_pairs((n, 8), (n, 8)) -> (n, 8)` do the hashing — one call per
    level for all queries — so the caller decides where it runs.  `dims`: [(width, height)] per matrix; `opened_values[q][m]`."""
    def req(cond, msg):
        if not cond:
            raise MerkleTreeError(msg)
    cap = np.asarray(cap, dtype=np.uint32).reshape(-1, 8)
    log_cap = cap.shape[0].bit_length() - 1
    req(len(dims) > 0 and cap.shape[0] == 1 << log_cap, "wrong batch size")
    logs = [_log2_ceil(int(h)) for _, h in dims]
    log_max = max(logs)
    req(log_cap <= log_max and min(logs) >= log_cap, "matrix heights do not fit the cap")
    req(len(opened_values) == len(indices), "wrong batch size")
    by_level = {}
    for m, lg in enumerate(logs):
        by_level.setdefault(lg, []).append(m)
    rows_at = [dict() for _ in dims]                                  # per matrix: reduced index -> opened row (must be unique)
    rep = {}
    for q, (i, rows) in enumerate(zip(indices, opened_values)):
        req(0 <= int(i) < (1 << log_max), "index out of bounds")
        req(len(rows) == len(dims), "wrong batch size")
        for m, (row, (w, _)) in enumerate(zip(rows, dims)):
            row = np.asarray(row, dtype=np.uint32).ravel()
            req(row.size == w, "wrong width")
            known = rows_at[m].setdefault(int(i) >> (log_max - logs[m]), row)
            req(known is row or np.array_equal(known, row), "two openings of one row disagree")
        rep.setdefault(int(i), q)
    nodes = sorted(rep)

    def level_digests(lg, node_ids):
        ms = by_level[lg]
        return hash_rows(np.stack([np.concatenate([rows_at[m][nid] for m in ms]) for nid in node_ids]))

    dig = np.asarray(level_digests(log_max, nodes), dtype=np.uint32).reshape(len(nodes), 8)
    pruned = np.asarray(pruned, dtype=np.uint32).reshape(-1, 8)
    k = 0
    for lvl in range(log_max, log_cap, -1):
        left, right, parents, j = [], [], [], 0
        while j < len(nodes):
            idx = nodes[j]
            if j + 1 < len(nodes) and nodes[j + 1] == (idx ^ 1):
                left.append(dig[j]); right.append(dig[j + 1]); j += 2
            else:
                req(k < pruned.shape[0], "multiproof is shorter than its frontier")
                sib = pruned[k]; k += 1
                if idx & 1:
                    left.append(sib); right.append(dig[j])
                else:
                    left.append(dig[j]); right.append(sib)
                j += 1
            parents.append(idx >> 1)
        dig = np.asarray(compress_pairs(np.array(left, dtype=np.uint32), np.array(right, dtype=np.uint32)), dtype=np.uint32).reshape(len(parents), 8)
        nodes = parents
        if (lvl - 1) in by_level:                                     # inject the matrices of this height
            inj = np.asarray(level_digests(lvl - 1, nodes), dtype=np.uint32).reshape(len(nodes), 8)
            dig = np.asarray(compress_pairs(dig, inj), dtype=np.uint32).reshape(len(nodes), 8)
    req(k == pruned.shape[0], "multiproof holds digests the frontier does not use")
    for idx, d in zip(nodes, dig):
        req(np.array_equal(cap[idx], d), "cap mismatch")


class MerkleTreeMmcs:
    """MerkleTreeMmcs<P, PW, H, C, 2, 8>.

    hash configurations (examples/src/types.rs:19-53, merkle-tree/benches/merkle_tree.rs:38):
      MerkleTreeMmcs.poseidon2(perm16)            leaf PaddingFreeSponge<Perm16,16,8,8>,  node TruncatedPermutation<Perm16,2,8,16>
      MerkleTreeMmcs.poseidon2(perm16, perm24)    leaf PaddingFreeSponge<Perm24,24,16,8>, node TruncatedPermutation<Perm16,2,8,16>
      MerkleTreeMmcs.keccak(field)                leaf SerializingHasher<PaddingFreeSponge<KeccakF,25,17,4>>, node CompressionFunctionFromHasher
      MerkleTreeMmcs.sha256(field)                leaf SerializingHasher<Sha256>, node CompressionFunctionFromHasher<Sha256, 2, 32>
      MerkleTreeMmcs.sha256(field, node="compress")  leaf SerializingHasher<Sha256>, node Sha256Compress
    """

    def __init__(self, field: Field, hash_kind: int, cap_height: int = 0, gpu: Optional[Gpu] = None, perms=()):
        self.field, self.hash_kind, self.cap_height = field, hash_kind, cap_height
        self.gpu = gpu or default_gpu()
        self.perms = perms

    @classmethod
    def poseidon2(cls, perm16: Poseidon2, perm24: Optional[Poseidon2] = None, cap_height: int = 0, gpu=None):
        assert perm16.width == 16 and (perm24 is None or perm24.width == 24)
        kind = _lib.HASH_POSEIDON2_W24 if perm24 is not None else _lib.HASH_POSEIDON2_W16
        return cls(perm16.field, kind, cap_height, gpu, tuple(p for p in (perm16, perm24) if p is not None))

    @classmethod
    def keccak(cls, field: Field, cap_height: int = 0, gpu=None):
        return cls(field, _lib.HASH_KECCAK, cap_height, gpu)

    @classmethod
    def sha256(cls, field: Field, cap_height: int = 0, gpu=None, node: str = "hasher"):
        """MerkleTreeMmcs<F, u8, SerializingHasher<Sha256>, C, 2, 32> (keccak-air/examples/prove_baby_bear_sha256*.rs): `node`
        "hasher" is C = CompressionFunctionFromHasher<Sha256, 2, 32>, "compress" is C = Sha256Compress.  Digests are [u8; 32], held
        as 8 words whose little-endian bytes are the digest's bytes."""
        kinds = {"hasher": _lib.HASH_SHA256, "compress": _lib.HASH_SHA256_COMPRESS}
        if node not in kinds:
            raise ValueError(f"unknown SHA-256 node compression {node!r} (\"hasher\" or \"compress\")")
        return cls(field, kinds[node], cap_height, gpu)

    # commit/src/mmcs.rs:42, merkle-tree/src/mmcs/batch.rs:42-64
    def commit(self, inputs: list):
        if len(inputs) == 0:
            raise _lib.P3GpuError("No matrices given?")
        for p in self.perms:
            p.upload(self.gpu)
        layers = self.gpu.merkle_commit(self.field.id, self.hash_kind, inputs)
        tree = MerkleTree(list(inputs), layers, [2] * (len(layers) - 1))
        eff = min(self.cap_height, max(tree.num_layers() - 1, 0))
        return tree.cap(eff), tree

    def commit_matrix(self, m):
        return self.commit([m])

    # commit/src/mmcs.rs:106
    def get_matrices(self, prover_data: MerkleTree):
        return list(prover_data.leaves)

    def get_max_height(self, prover_data: MerkleTree):
        return max(int(m.shape[0]) for m in prover_data.leaves)

    # merkle-tree/src/mmcs/batch.rs:75-121
    def open_batch(self, index: int, prover_data: MerkleTree):
        max_height = self.get_max_height(prover_data)
        if index >= max_height:
            raise IndexError(f"index {index} out of bounds for height {max_height}")
        log_max = _log2_ceil(max_height)
        openings = []
        for m in prover_data.leaves:
            bits_reduced = log_max - _log2_ceil(int(m.shape[0]))
            openings.append(_host(m[index >> bits_reduced]))
        nl = prover_data.num_layers()
        eff = min(self.cap_height, max(nl - 1, 0))
        proof, idx = [], index
        for layer_idx in range(nl - 1 - eff):
            proof.append(_host(prover_data.digest_layers[layer_idx][(idx ^ 1):(idx ^ 1) + 1])[0])
            idx >>= 1
        return openings, proof

    # commit/src/mmcs.rs:173 / merkle-tree/src/mmcs/mod.rs:276-428 (without the path pruning, which is a host-side re-encoding)
    def open_multi_batch(self, indices, prover_data: MerkleTree):
        """open_batch for many indices at once.  Returns (openings: per matrix an (n, width) uint32 array, paths: (n, path_len, 8)
        uint32 array of sibling digests, bottom-up).  Device-resident prover data is gathered by two small kernels
        (csrc/query.cu) and copied back once per matrix."""
        import ctypes as C
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        n = int(idx.size)
        max_height = self.get_max_height(prover_data)
        if n and int(idx.max()) >= max_height:
            raise IndexError(f"index {int(idx.max())} out of bounds for height {max_height}")
        log_max = _log2_ceil(max_height)
        gpu = self.gpu
        openings = []
        for m in prover_data.leaves:
            shift = log_max - _log2_ceil(int(m.shape[0]))
            if _is_torch(m) and m.is_cuda:
                gpu._use_torch_stream()
                out = gpu._empty((n, int(m.shape[1])))
                _lib.check(gpu.L.p3gpu_gather_rows_dev(gpu.h, m.data_ptr(), int(m.shape[0]), int(m.shape[1]), idx.ctypes.data, n, shift, out.data_ptr()))
                openings.append(_host(out))
            else:
                openings.append(np.array(_host(m)[idx >> shift], dtype=np.uint32))
        nl = prover_data.num_layers()
        eff = min(self.cap_height, max(nl - 1, 0))
        path_len = nl - 1 - eff
        layers = prover_data.digest_layers
        if path_len == 0 or n == 0:
            return openings, np.zeros((n, path_len, 8), dtype=np.uint32)
        if _is_torch(layers[0]) and layers[0].is_cuda:
            lens = (C.c_size_t * nl)(*[int(l.shape[0]) for l in layers])
            base, off = layers[0].data_ptr(), 0
            for l in layers:                                             # all layers of a commit are slices of one device buffer
                assert l.data_ptr() == base + off * 32, "digest layers are not contiguous"
                off += int(l.shape[0])
            gpu._use_torch_stream()
            out = gpu._empty((n, path_len, 8))
            _lib.check(gpu.L.p3gpu_merkle_paths_dev(gpu.h, base, lens, nl, path_len, idx.ctypes.data, n, 0, out.data_ptr()))
            return openings, _host(out)
        paths = np.zeros((n, path_len, 8), dtype=np.uint32)
        for l in range(path_len):
            paths[:, l] = _host(layers[l])[(idx >> l) ^ 1]
        return openings, paths

    # ---- verifier side: batch hashing on the device (SURVEY 8f rank 4)
    def hash_rows(self, rows):
        """Leaf digests of n rows ((n, w) Montgomery words) — the leaf kernel on an n-row matrix."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        for p in self.perms:
            p.upload(self.gpu)
        return _host(self.gpu.merkle_commit(self.field.id, self.hash_kind, [rows])[0])[: rows.shape[0]]

    def compress_pairs(self, left, right):
        """compress([left[i], right[i]]) for n pairs: the node kernel on the interleaved digests (one tree level)."""
        left = np.asarray(left, dtype=np.uint32).reshape(-1, 8)
        inter = np.empty((2 * left.shape[0], 8), dtype=np.uint32)
        inter[0::2] = left; inter[1::2] = np.asarray(right, dtype=np.uint32).reshape(-1, 8)
        for p in self.perms:
            p.upload(self.gpu)
        import torch
        dev = torch.from_numpy(inter.view(np.int32)).to(f"cuda:{self.gpu.device}")
        return _host(self.gpu.merkle_from_digests(self.field.id, self.hash_kind, dev)[1])[: left.shape[0]]

    # commit/src/mmcs.rs:190-199, merkle-tree/src/mmcs/batch.rs:286-296
    def verify_multi_batch(self, commit, dimensions, indices, opened_values, proof):
        """Raises MerkleTreeError.  `dimensions`: [(width, height)]; `proof`: the pruned multiproof (k, 8)."""
        verify_multi_batch_with(self.hash_rows, self.compress_pairs, commit, dimensions, indices, opened_values, proof)

    # merkle-tree/src/mmcs/batch.rs:275-284, mmcs/mod.rs:276-428: the wire form of a multi-opening
    def open_multi_batch_pruned(self, indices, prover_data: MerkleTree):
        """Returns (opened_values[query][matrix] = row, pruned multiproof (k, 8)): the device gathers of `open_multi_batch`
        followed by the host-side re-encoding `prune_paths`."""
        openings, paths = self.open_multi_batch(indices, prover_data)
        opened_values = [[openings[m][q] for m in range(len(openings))] for q in range(len(indices))]
        return opened_values, prune_paths(indices, paths)
