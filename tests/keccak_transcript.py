"""Restatement of the Keccak configuration's transcript — TEST INFRASTRUCTURE, never importable from the product.

    keccak256            Keccak256Hash (keccak/src/lib.rs:100-130, tiny-keccak v256) on the oracle's Keccak-f: rate 136 bytes, padding
                         0x01 ... 0x80, the whole message hashed at once
    HashChallenger       challenger/src/hash_challenger.rs over bytes, literally: an input buffer that keeps every observed byte, an
                         output buffer the samples pop from the end of, flush = hash the whole input buffer
    SerializingChallenger32
                         challenger/src/serializing_challenger.rs on top, with the surface of plonky3_b200.challenger
                         (Montgomery words in and out; observe_cap takes digests as words whose bytes are observed)

The device keeps a running Keccak state and a partial block instead of the input buffer (csrc/challenger.cu); this module does not,
so the two agree only if that is equivalent.  `grind` is the sequential search from 0, which returns the smallest witness."""
import numpy as np

from oracle import p3_oracle as O


def _absorb(state, blocks: bytes):
    for off in range(0, len(blocks), 136):
        state = state.copy()
        state[:17] ^= np.frombuffer(blocks[off:off + 136], dtype="<u8")
        state = O.keccak_f(state)
    return state


def keccak256_finish(state, tail: bytes) -> bytes:
    """The rest of keccak256 after `state` absorbed whole blocks: the tail, the padding, the squeeze."""
    msg = bytearray(tail)
    msg.append(0x01)
    msg += bytes((-len(msg)) % 136)
    msg[-1] |= 0x80
    return _absorb(state, bytes(msg))[:4].astype("<u8").tobytes()


def keccak256(msg: bytes) -> bytes:
    return keccak256_finish(np.zeros(25, dtype=np.uint64), msg)


class HashChallenger:
    """HashChallenger<u8, H, 32>; `hasher(bytes) -> 32 bytes`."""

    def __init__(self, initial_state=b"", hasher=keccak256):
        self.input, self.output, self.hasher = bytearray(initial_state), bytearray(), hasher

    def clone(self):
        c = HashChallenger(self.input, self.hasher)
        c.output = bytearray(self.output)
        return c

    def observe_bytes(self, bs):
        for b in bytes(bs):
            self.output.clear()                                   # any buffered output is now invalid
            self.input.append(b)

    def flush(self):
        out = self.hasher(bytes(self.input))
        assert len(out) == 32
        self.input = bytearray(out)                               # chaining value
        self.output = bytearray(out)

    def sample_byte(self) -> int:
        if not self.output:
            self.flush()
        return self.output.pop()

    def sample_array(self, n: int) -> bytes:
        return bytes(self.sample_byte() for _ in range(n))


class SerializingChallenger32:
    """SerializingChallenger32<F, HashChallenger<u8, H, 32>> for one plonky3_b200.field.Field."""

    def __init__(self, field, inner: HashChallenger = None):
        self.field, self.inner = field, inner if inner is not None else HashChallenger()

    @classmethod
    def from_hasher(cls, field, initial_state=b"", hasher=keccak256):
        return cls(field, HashChallenger(initial_state, hasher))

    def clone(self):
        return SerializingChallenger32(self.field, self.inner.clone())

    # ---- CanObserve
    def observe(self, word: int):                                # F: the canonical value's 4 little-endian bytes
        self.inner.observe_bytes(int(self.field.from_monty(int(word))).to_bytes(4, "little"))

    def observe_slice(self, words):
        for w in _words(words):
            self.observe(int(w))

    def observe_canonical(self, x: int): self.observe(self.field.to_monty(int(x)))
    def observe_algebra_slice(self, ys): self.observe_slice(ys)

    def observe_cap(self, cap):                                  # MerkleCap<F, [u64; 4]>: each u64's 8 little-endian bytes
        self.inner.observe_bytes(_words(cap).astype("<u4").tobytes())

    # ---- CanSample
    def _u32(self) -> int:
        return int.from_bytes(self.inner.sample_array(4), "little")

    def sample(self) -> int:
        while True:
            v = self._u32() & 0x7FFFFFFF                           # (1 << log2_ceil(p)) - 1
            if v < self.field.P:
                return self.field.to_monty(v)

    def sample_many(self, n: int) -> np.ndarray: return np.array([self.sample() for _ in range(n)], dtype=np.uint32)
    def sample_algebra_element(self) -> np.ndarray: return self.sample_many(4)

    def sample_bits(self, bits: int) -> int:
        assert (1 << bits) < self.field.P, "requested bit count must fit within the field order"
        return self._u32() & ((1 << bits) - 1)

    # ---- GrindingChallenger
    def check_witness(self, bits: int, word: int) -> bool:
        if bits == 0:
            return True
        self.observe(word)
        return self.sample_bits(bits) == 0

    def grind(self, bits: int) -> int:
        """The smallest canonical witness, as a Montgomery word; observed and its sample consumed.  With Keccak-256 the whole
        blocks of the input buffer are hashed once and each candidate only finishes the hash (the candidate's first sampled u32
        is the digest's last 4 bytes, popped last-first); any other hasher runs check_witness on a clone per candidate."""
        assert (1 << bits) < self.field.P, "requested bit count must fit within the field order"
        if bits == 0:
            return 0
        mask = (1 << bits) - 1
        if self.inner.hasher is keccak256:
            buf = bytes(self.inner.input)
            full = len(buf) - len(buf) % 136
            mid = _absorb(np.zeros(25, dtype=np.uint64), buf[:full])
            valid = lambda w: int.from_bytes(keccak256_finish(mid, buf[full:] + w.to_bytes(4, "little"))[28:][::-1], "little") & mask == 0
        else:
            valid = lambda w: self.clone().check_witness(bits, self.field.to_monty(w))
        for w in range(self.field.P):
            if valid(w):
                word = self.field.to_monty(w)
                assert self.check_witness(bits, word)
                return word
        raise AssertionError("failed to find witness")


def _words(a) -> np.ndarray:
    import torch
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().contiguous().numpy().view(np.uint32)
    return np.ascontiguousarray(a, dtype=np.uint32).ravel()


# ------------------------------------------------------------------------------------------------------------------
# The Keccak configuration's prove driver on the oracle-backed stand-in device (tests/mock_device.py): the product's host code
# (uni_stark.prove, the PCS, FRI, the Keccak MMCS's host side, the wire form) with every device call answered by the oracle and the
# transcript by the restatement above.  The GPU suite checks that the real kernels write the same bytes.
def p2_air_setup(field, seed: int = 1):
    """The example binary's AIR round constants (SmallRng seed 1, examples/examples/prove_prime_field_31.rs:115)."""
    rng = O.SmallRng(seed)
    return O.air_from_rng(field.id, rng)


def p2_round_constants(oair):
    from plonky3_b200.uni_stark import RoundConstants
    return RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p], np.array(oair.end).reshape(4, 16))


def p2_inputs(field, log_rows: int):
    return O.SmallRng(1).field(field.id, (8 << log_rows) * 16).reshape(-1, 16)


def keccak_mock_config(field, gpu, num_queries: int, pow_bits: int, cap_height: int = 3):
    """KeccakStarkConfig's shape on a stand-in device: Keccak MMCS with cap height 3, new_benchmark_high_arity's FRI parameters (with
    the query count and proof-of-work bits given), the restated transcript."""
    from types import SimpleNamespace
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    mmcs = MerkleTreeMmcs.keccak(field, cap_height=cap_height, gpu=gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(field, gpu), mmcs, FriParameters(1, 0, 3, num_queries, 0, pow_bits, mmcs))
    return SimpleNamespace(pcs=pcs, digest_codec="u64x4", initialise_challenger=lambda: SerializingChallenger32.from_hasher(field))


def verifier_config(field, num_queries: int, pow_bits: int, log_blowup: int = 1, log_final_poly_len: int = 0, max_log_arity: int = 3):
    """plonky3_b200.verifier's configuration with oracle stand-ins: Keccak MMCS hashing by the oracle, the restated transcript."""
    from types import SimpleNamespace
    import stark_verify as V
    from plonky3_b200.fri import FriParameters
    mmcs = V.OracleMmcs(O.keccak_hasher())
    fri = FriParameters(log_blowup, log_final_poly_len, max_log_arity, num_queries, 0, pow_bits, mmcs)
    return SimpleNamespace(pcs=SimpleNamespace(fri=fri, mmcs=mmcs, dft=SimpleNamespace(field=field)), digest_codec="u64x4",
                           initialise_challenger=lambda: SerializingChallenger32.from_hasher(field))


def mock_prove_p2(field, log_rows: int, num_queries: int, pow_bits: int):
    """The config-5 AIR (vectorised Poseidon2, 8 permutations a row) over 2^log_rows rows, proved on the stand-in device.  Returns
    (proof, air).  The caller stubs torch.cuda.synchronize (the driver's span timers)."""
    import mock_device as M
    import torch
    from plonky3_b200.uni_stark import VectorizedPoseidon2Air, prove
    gpu = M.MockGpu()
    config = keccak_mock_config(field, gpu, num_queries, pow_bits)
    air = VectorizedPoseidon2Air(field, p2_round_constants(p2_air_setup(field)), gpu)
    trace = air.generate_trace_rows(torch.from_numpy(p2_inputs(field, log_rows).view(np.int32)))
    return prove(config, air, trace), air
