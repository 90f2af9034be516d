"""The SHA-256 configurations restated on the host with hashlib — TEST INFRASTRUCTURE, never importable from the product.

    sha256 / hash_rows      Sha256 and SerializingHasher<Sha256>: a row's bytes are its Montgomery words little-endian
    compress_pairs          CompressionFunctionFromHasher<Sha256, 2, 32> ("hasher": SHA-256 of the 64 bytes) or Sha256Compress
                            ("compress": one raw compression from the IV, by tests/sha256_air_oracle.compress)
    merkle_tree             MerkleTree::new over those (merkle-tree/src/merkle_tree.rs), layers as (n, 8) words
    HashMmcs                the verifier-side MMCS surface (hash_rows / compress_pairs / verify_multi_batch) on the above
    transcript              tests/keccak_transcript.SerializingChallenger32 with hashlib's SHA-256 as the hasher
    with_sha256             a stand-in device (tests/mock_device.py) answering the two SHA-256 hash kinds with merkle_tree

A digest is held as 8 words whose little-endian bytes are the digest's bytes, as the device holds it."""
import hashlib

import numpy as np

import keccak_transcript as K
import mock_device as M
import sha256_air_oracle as SO
from plonky3_b200 import _lib

NODES = {_lib.HASH_SHA256: "hasher", _lib.HASH_SHA256_COMPRESS: "compress"}
IV = np.array(SO.IV, dtype=np.uint32)


def sha256(msg: bytes) -> bytes:
    return hashlib.sha256(bytes(msg)).digest()


def words(d: bytes) -> np.ndarray:
    return np.frombuffer(d, dtype="<u4").astype(np.uint32)


def hash_rows(rows) -> np.ndarray:
    """(n, w) Montgomery words -> (n, 8) leaf digests."""
    rows = np.ascontiguousarray(np.asarray(rows, dtype=np.uint32).reshape(len(rows), -1)).astype("<u4")
    out = np.empty((rows.shape[0], 8), dtype=np.uint32)
    for i in range(rows.shape[0]):
        out[i] = words(sha256(rows[i].tobytes()))
    return out


def compress_pairs(left, right, node: str) -> np.ndarray:
    left = np.asarray(left, dtype=np.uint32).reshape(-1, 8)
    right = np.asarray(right, dtype=np.uint32).reshape(-1, 8)
    both = np.ascontiguousarray(np.hstack([left, right])).astype("<u4")
    if node == "hasher":
        out = np.empty((both.shape[0], 8), dtype=np.uint32)
        for i in range(both.shape[0]):
            out[i] = words(sha256(both[i].tobytes()))
        return out
    assert node == "compress", node
    block = both.astype(np.uint32).byteswap()                     # big-endian message words
    st = SO.compress(np.tile(IV, (block.shape[0], 1)), block)
    return np.ascontiguousarray(st, dtype=np.uint32).byteswap()


def _next_pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _padded(raw):
    return raw if raw <= 1 else (raw + 1) // 2 * 2


def merkle_tree(mats, node: str):
    """MerkleTree::new with arity 2 (merkle_tree.rs:95-178, first_digest_layer, compress, compress_and_inject): the tallest
    matrices' rows concatenated make the leaves; shorter matrices are injected at the layer of their padded height."""
    mats = [np.asarray(m, dtype=np.uint32).reshape(m.shape[0], -1) for m in mats]
    order = sorted(range(len(mats)), key=lambda i: -mats[i].shape[0])
    max_h = mats[order[0]].shape[0]
    nxt = 0
    while nxt < len(order) and mats[order[nxt]].shape[0] == max_h:
        nxt += 1
    cur = np.zeros((_padded(max_h), 8), dtype=np.uint32)
    cur[:max_h] = hash_rows(np.hstack([mats[i] for i in order[:nxt]]))
    layers = [cur]
    while cur.shape[0] > 1:
        raw = cur.shape[0] // 2
        begin = nxt
        while nxt < len(order) and _next_pow2(mats[order[nxt]].shape[0]) == _next_pow2(raw):
            nxt += 1
        out = np.zeros((_padded(raw), 8), dtype=np.uint32)
        out[:raw] = compress_pairs(cur[0:2 * raw:2], cur[1:2 * raw:2], node)
        if nxt > begin:
            inj_h = mats[order[begin]].shape[0]
            inj = np.zeros((raw, 8), dtype=np.uint32)
            inj[:inj_h] = hash_rows(np.hstack([mats[i] for i in order[begin:nxt]]))
            out[:raw] = compress_pairs(out[:raw], inj, node)
        layers.append(out)
        cur = out
    return layers


def cap(layers, cap_height):
    nl = len(layers)
    eff = min(cap_height, max(nl - 1, 0))
    layer = layers[nl - 1 - eff]
    return layer[: min(1 << eff, len(layer))].copy()


class HashMmcs:
    """The verifier-side surface of plonky3_b200.merkle_tree.MerkleTreeMmcs with hashlib's SHA-256."""

    def __init__(self, node: str):
        self.node = node

    def hash_rows(self, rows): return hash_rows(rows)
    def compress_pairs(self, left, right): return compress_pairs(left, right, self.node)

    def verify_multi_batch(self, commit, dims, indices, opened_values, proof):
        from plonky3_b200.merkle_tree import verify_multi_batch_with
        verify_multi_batch_with(self.hash_rows, self.compress_pairs, commit, dims, indices, opened_values, proof)


def transcript(field, initial_state=b""):
    """SerializingChallenger32<F, HashChallenger<u8, Sha256, 32>>, restated."""
    return K.SerializingChallenger32.from_hasher(field, initial_state, sha256)


def fri_commit_phase(f, node, cap_height, vec, log_blowup, log_final_poly_len, max_log_arity, betas):
    """The FRI commit phase of one input vector with given betas (fri/src/prover.rs:192-286), folding by the C oracle and committing
    by merkle_tree.  Returns (caps, log_arities, final folded vector)."""
    from oracle import p3_oracle as O
    folded = np.asarray(vec, dtype=np.uint32)
    caps, arities = [], []
    log_final = log_blowup + log_final_poly_len
    k = 0
    while folded.shape[0] > (1 << log_final):
        la = O.compute_log_arity_for_round(int(np.log2(folded.shape[0])), None, log_final, max_log_arity)
        arities.append(la)
        caps.append(cap(merkle_tree([folded.reshape(folded.shape[0] >> la, (1 << la) * 4)], node), cap_height))
        folded = O.fold_matrix(f, folded, la, np.asarray(betas[k], dtype=np.uint32))
        k += 1
    return caps, arities, folded


def verifier_config(field, node, fri):
    """plonky3_b200.verifier's configuration with hashlib stand-ins: the SHA-256 MMCS and the restated transcript.  `fri`: the
    FriParameters fields (log_blowup, log_final_poly_len, max_log_arity, num_queries, commit_pow_bits, query_pow_bits)."""
    from types import SimpleNamespace
    from plonky3_b200.fri import FriParameters
    mmcs = HashMmcs(node)
    params = FriParameters(*fri, mmcs)
    return SimpleNamespace(pcs=SimpleNamespace(fri=params, mmcs=mmcs, dft=SimpleNamespace(field=field)), digest_codec="u8x32",
                           initialise_challenger=lambda: transcript(field))


def with_sha256(base=M.MockGpu):
    """A subclass of an oracle-backed stand-in device (tests/mock_device.MockGpu or a subclass of it) that also answers the two
    SHA-256 hash kinds, with merkle_tree."""

    class MockShaGpu(base):
        def merkle_commit(self, field, hash_kind, mats):
            if hash_kind not in NODES:
                return super().merkle_commit(field, hash_kind, mats)
            self._note("merkle_commit")
            return merkle_tree([M._n(m) for m in mats], NODES[hash_kind])
    return MockShaGpu


def mock_config(field, gpu, node, fri, cap_height):
    """Sha256StarkConfig's shape on a stand-in device, with the restated transcript."""
    from types import SimpleNamespace
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    mmcs = MerkleTreeMmcs.sha256(field, cap_height=cap_height, gpu=gpu, node=node)
    pcs = TwoAdicFriPcs(Radix2DitParallel(field, gpu), mmcs, FriParameters(*fri, mmcs))
    return SimpleNamespace(pcs=pcs, digest_codec="u8x32", initialise_challenger=lambda: transcript(field))
