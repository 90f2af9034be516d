"""Wire form of a uni-stark proof: what `postcard::to_allocvec(&Proof<SC>)` writes for
SC = StarkConfig<TwoAdicFriPcs<Val, Dft, MerkleTreeMmcs<.., 2, 8>, ExtensionMmcs<..>>, BinomialExtensionField<Val, 4>, ..>
(uni-stark/tests/fib_air.rs:401-412), so that a proof made on the GPU is read by the reference's verifier with
`postcard::from_bytes` and vice versa.  Host-side re-encoding only; no field arithmetic happens here.

Layout = serde declaration order, postcard rules:
  Proof            { commitments, opened_values, opening_proof, degree_bits: usize }                 uni-stark/src/proof.rs:19-26
  Commitments      { trace: MerkleCap, quotient_chunks: MerkleCap, random: Option<..> }              proof.rs:44-49
  OpenedValues     { trace_local: Vec<EF>, trace_next: Option<Vec<EF>>, preprocessed_local: Option, preprocessed_next: Option,
                     quotient_chunks: Vec<Vec<EF>>, random: Option }                                 proof.rs:51-62
  FriProof         { commit_phase_commits: Vec<MerkleCap>, commit_pow_witnesses: Vec<F>, input_openings: Vec<BatchMultiOpening>,
                     commit_phase_openings: Vec<CommitPhaseMultiStep>, final_poly: Vec<EF>, query_pow_witness: F }   fri/src/proof.rs:12-24
  BatchMultiOpening{ opened_values: Vec<Vec<Vec<F>>> (query, matrix, column), opening_proof: PrunedMerklePaths }      fri/src/proof.rs:68-75
  CommitPhaseMultiStep { log_arity: u8, sibling_values: Vec<Vec<EF>>, opening_proof: PrunedMerklePaths }              fri/src/proof.rs:33-44
  PrunedMerklePaths{ sibling_hashes: Vec<[F; 8]> }                                                   merkle-tree/src/pruning.rs:83-89
  MerkleCap = Vec<[F; 8]>;  Vec = varint length + items;  Option = tag byte;  usize = varint;  u8 = one byte;  arrays carry no length;
  F = the 4 little-endian bytes of the Montgomery word (monty-31/src/monty_31.rs:167-179);  EF = 4 F.
Digests (caps, FRI commit-phase caps, pruned-path sibling hashes) take one of two codecs.  DIGEST_F8, the default: [F; 8] (the
Poseidon2 MMCS), 8 Montgomery words.  DIGEST_U64X4: [u64; 4] (the Keccak MMCS, examples/src/types.rs:19-35), held as 8 words
(lo, hi of each u64) and written as 4 postcard varints of at most 10 bytes each.  DIGEST_U8X32: [u8; 32] (the SHA-256 MMCS,
keccak-air/examples/prove_baby_bear_sha256*.rs), held as 8 words whose little-endian bytes are the digest's bytes and written as
those 32 raw bytes (a postcard array carries no length; the Vec around it keeps its varint length).
Pinned byte for byte against the reference's committed proof fixture (tests/golden/uni_stark_two_adic_v1.json `postcard_hex`)."""
from __future__ import annotations

import numpy as np

from .merkle_tree import prune_paths

DIGEST_F8, DIGEST_U64X4, DIGEST_U8X32 = "f8", "u64x4", "u8x32"
DIGEST_CODECS = (DIGEST_F8, DIGEST_U64X4, DIGEST_U8X32)


def _varint(n: int) -> bytes:
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _words(a) -> bytes:
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint32)).astype("<u4").tobytes()


def _vec_of(a, width: int) -> bytes:
    """Vec<[F; width]> (width = 8: digests / caps, 4: extension elements)."""
    a = np.asarray(a, dtype=np.uint32).reshape(-1, width)
    return _varint(a.shape[0]) + _words(a)


def _vec_of_digests(a, digest: str) -> bytes:
    """Vec<digest>: a cap or a pruned path's sibling hashes, (n, 8) words."""
    if digest in (DIGEST_F8, DIGEST_U8X32):                        # [u8; 32]: the words' own bytes, no range to respect
        return _vec_of(a, 8)
    if digest != DIGEST_U64X4:
        raise ValueError(f"unknown digest codec {digest!r}")
    a = np.asarray(a, dtype=np.uint32).reshape(-1, 8).astype(np.uint64)
    lanes = a[:, 0::2] | (a[:, 1::2] << np.uint64(32))
    return _varint(a.shape[0]) + b"".join(_varint(int(v)) for v in lanes.ravel())


def _option_vec_ef(a) -> bytes:
    return b"\x00" if a is None else b"\x01" + _vec_of(a, 4)


def proof_to_postcard(proof, digest: str = DIGEST_F8) -> bytes:
    """`proof`: plonky3_b200.uni_stark.Proof (non-ZK).  `digest`: DIGEST_F8, DIGEST_U64X4 or DIGEST_U8X32, the configuration's
    digest type."""
    vd = lambda a: _vec_of_digests(a, digest)
    out = bytearray()
    out += vd(proof.trace_commit) + vd(proof.quotient_commit) + b"\x00"
    out += _vec_of(proof.trace_local, 4) + _option_vec_ef(proof.trace_next)
    out += _option_vec_ef(getattr(proof, "preprocessed_local", None)) + _option_vec_ef(getattr(proof, "preprocessed_next", None))
    out += _varint(len(proof.quotient_chunks)) + b"".join(_vec_of(c, 4) for c in proof.quotient_chunks) + b"\x00"
    out += _varint(len(proof.commit_phase_commits)) + b"".join(vd(c) for c in proof.commit_phase_commits)
    out += _varint(len(proof.commit_pow_witnesses)) + _words(np.array(proof.commit_pow_witnesses, dtype=np.uint32))
    assert len(proof.input_opening_indices) == len(proof.input_openings) and len(proof.commit_phase_indices) == len(proof.commit_phase_openings)
    out += _varint(len(proof.input_openings))
    for (rows, paths), idx in zip(proof.input_openings, proof.input_opening_indices):
        out += _varint(len(idx))
        if len(idx):                                              # all queries have the same byte layout: assemble them as one (n, bytes) block
            n = len(idx)
            parts = [np.tile(np.frombuffer(_varint(len(rows)), dtype=np.uint8), (n, 1))]
            for m in rows:
                m = np.ascontiguousarray(np.asarray(m, dtype=np.uint32).reshape(n, -1)).astype("<u4")
                parts.append(np.tile(np.frombuffer(_varint(m.shape[1]), dtype=np.uint8), (n, 1)))
                parts.append(m.view(np.uint8).reshape(n, -1))
            out += np.hstack(parts).tobytes()
        out += vd(prune_paths(idx, paths))
    out += _varint(len(proof.commit_phase_openings))
    for (log_arity, siblings, paths), idx in zip(proof.commit_phase_openings, proof.commit_phase_indices):
        out += bytes([log_arity]) + _varint(len(idx))
        if len(idx):
            sib = np.ascontiguousarray(np.asarray(siblings, dtype=np.uint32).reshape(len(idx), -1)).astype("<u4")      # (n, (arity - 1) * 4)
            pre = np.tile(np.frombuffer(_varint(sib.shape[1] // 4), dtype=np.uint8), (len(idx), 1))
            out += np.hstack([pre, sib.view(np.uint8).reshape(len(idx), -1)]).tobytes()
        out += vd(prune_paths(idx, paths))
    out += _vec_of(proof.final_poly, 4) + _words([proof.query_pow_witness]) + _varint(proof.degree_bits)
    return bytes(out)


class _Reader:
    def __init__(self, data: bytes, prime=None, digest: str = DIGEST_F8):
        if digest not in DIGEST_CODECS:
            raise ValueError(f"unknown digest codec {digest!r}")
        self.b, self.pos, self.prime, self.digest = data, 0, prime, digest

    def varint(self) -> int:
        r = s = 0
        while True:
            if self.pos >= len(self.b):
                raise ValueError("truncated proof")
            c = self.b[self.pos]; self.pos += 1
            r |= (c & 0x7F) << s; s += 7
            if c < 0x80:
                return r

    def u64(self) -> int:
        """A postcard u64: at most 10 varint bytes, the value below 2^64."""
        r = 0
        for k in range(10):
            if self.pos >= len(self.b):
                raise ValueError("truncated proof")
            c = self.b[self.pos]; self.pos += 1
            r |= (c & 0x7F) << (7 * k)
            if c < 0x80:
                if r >= 1 << 64:
                    raise ValueError("u64 varint out of range")
                return r
        raise ValueError("u64 varint longer than 10 bytes")

    def digests(self) -> np.ndarray:
        """Vec<digest> as (n, 8) words."""
        if self.digest == DIGEST_F8:
            return self.vec_of(8)
        if self.digest == DIGEST_U8X32:                             # 32 raw bytes each, any values
            n = self.varint()
            if 32 * n > len(self.b) - self.pos:
                raise ValueError("truncated proof")
            a = np.frombuffer(self.b, dtype="<u4", count=8 * n, offset=self.pos).astype(np.uint32).reshape(n, 8)
            self.pos += 32 * n
            return a
        n = self.varint()
        if n > len(self.b) - self.pos:                              # every u64 takes at least one byte
            raise ValueError("truncated proof")
        lanes = [self.u64() for _ in range(4 * n)]
        out = np.empty((n, 8), dtype=np.uint32)
        for k, v in enumerate(lanes):
            out[k // 4, 2 * (k % 4)] = v & 0xFFFFFFFF
            out[k // 4, 2 * (k % 4) + 1] = v >> 32
        return out

    def byte(self) -> int:
        if self.pos >= len(self.b):
            raise ValueError("truncated proof")
        self.pos += 1
        return self.b[self.pos - 1]

    def words(self, n: int) -> np.ndarray:
        if self.pos + 4 * n > len(self.b):
            raise ValueError("truncated proof")
        a = np.frombuffer(self.b, dtype="<u4", count=n, offset=self.pos).astype(np.uint32)
        self.pos += 4 * n
        if self.prime is not None and n and int(a.max()) >= self.prime:
            raise ValueError("Value is out of range")               # MontyField31::deserialize (monty-31/src/monty_31.rs:181-196)
        return a

    def vec_of(self, width: int) -> np.ndarray:
        n = self.varint()
        return self.words(n * width).reshape(n, width)

    def option_vec_ef(self):
        tag = self.byte()
        if tag > 1:
            raise ValueError("bad Option tag")
        return self.vec_of(4) if tag else None


def proof_from_postcard(data: bytes, prime=None, digest: str = DIGEST_F8) -> dict:
    """The inverse: every field of the wire proof as arrays of Montgomery words (pruned multiproofs are left pruned — the
    verifier consumes them against its own query indices).  With `prime` given, words >= prime are rejected as the reference's
    deserialiser rejects them (one field element has one encoding).  Digests (DIGEST_U64X4: 4 u64 varints, DIGEST_U8X32: 32 bytes)
    come back as (n, 8) words either way.  Raises ValueError on malformed input."""
    r = _Reader(data, prime, digest)
    p = {"trace_commit": r.digests(), "quotient_commit": r.digests()}
    if r.byte() != 0:
        raise ValueError("ZK (random) commitments are not supported")
    p["trace_local"] = r.vec_of(4)
    p["trace_next"] = r.option_vec_ef()
    p["preprocessed_local"] = r.option_vec_ef()
    p["preprocessed_next"] = r.option_vec_ef()
    p["quotient_chunks"] = [r.vec_of(4) for _ in range(r.varint())]
    if r.byte() != 0:
        raise ValueError("ZK (random) openings are not supported")
    p["commit_phase_commits"] = [r.digests() for _ in range(r.varint())]
    p["commit_pow_witnesses"] = [int(v) for v in r.words(r.varint())]
    p["input_openings"] = []
    for _ in range(r.varint()):
        ov = [[r.words(r.varint()) for _ in range(r.varint())] for _ in range(r.varint())]
        p["input_openings"].append({"opened_values": ov, "proof": r.digests()})
    p["commit_phase_openings"] = []
    for _ in range(r.varint()):
        la = r.byte()
        sv = [r.vec_of(4) for _ in range(r.varint())]
        p["commit_phase_openings"].append({"log_arity": la, "sibling_values": sv, "proof": r.digests()})
    p["final_poly"] = r.vec_of(4)
    p["query_pow_witness"] = int(r.words(1)[0])
    p["degree_bits"] = r.varint()
    if r.pos != len(data):
        raise ValueError("trailing bytes after the proof")
    return p
