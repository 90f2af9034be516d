"""DuplexChallenger (challenger/src/duplex_challenger.rs:60-300) + GrindingChallenger::grind (grinding_challenger.rs:100-232) with the
sponge resident on the GPU (csrc/challenger.cu): caps and opened values produced on the device are absorbed there; only sampled
challenges come back.  SerializingChallenger32 over a Keccak-256 or SHA-256 HashChallenger is the same on the device for the Keccak
and SHA-256 configurations.  Protocol plumbing of the prove driver (uni_stark.py), mirroring the reference's method names."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check
from .field import Field
from .gpu import _is_torch
from .poseidon2 import Poseidon2


class _DeviceChallenger:
    """The method surface both device transcripts share, behind one C handle; a subclass only creates the handle.  Values in and
    out are Montgomery words, as everywhere else in the prover."""

    def _create(self, new):
        """`new(out)`: a C call writing the new handle to `out`."""
        self.h = None
        h = C.c_void_p()
        self.gpu._use_torch_stream()
        check(new(C.byref(h)))
        self.h = h

    def __del__(self):
        try:
            if getattr(self, "h", None) and self.gpu.h:
                self.gpu.L.p3gpu_challenger_free(self.gpu.h, self.h)
                self.h = None
        except Exception:
            pass

    def clone(self):
        c = object.__new__(type(self))
        c.__dict__.update(self.__dict__)
        c._create(lambda out: self.gpu.L.p3gpu_challenger_clone(self.gpu.h, self.h, out))
        return c

    # ---- CanObserve
    def observe_slice(self, values):
        """Montgomery words (field elements); a CUDA int32 tensor is absorbed on the device without a copy."""
        self.gpu._use_torch_stream()
        if _is_torch(values) and values.is_cuda:
            v = values.contiguous()
            check(self.gpu.L.p3gpu_challenger_observe_dev(self.gpu.h, self.h, v.data_ptr(), v.numel()))
            self._keep = v
            return
        v = _host_words(values)
        check(self.gpu.L.p3gpu_challenger_observe(self.gpu.h, self.h, v.ctypes.data, v.size))

    def observe(self, value: int): self.observe_slice(np.array([value], dtype=np.uint32))
    def observe_canonical(self, x: int): self.observe(self.field.to_monty(x))           # Val::from_u8 / from_usize
    def observe_algebra_slice(self, ys): self.observe_slice(ys)                        # EF4 = 4 base coefficients in order

    def observe_cap(self, cap):
        """A Merkle cap's digests as the MMCS commits them: [F; 8] digests element by element (the duplex transcript); [u64; 4] or
        [u8; 32] digests, held as 8 words, as their 32 bytes (the byte transcripts)."""
        v = _host_words(cap)
        self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_challenger_observe_digest(self.gpu.h, self.h, v.ctypes.data, v.size))

    # ---- CanSample
    def sample_many(self, n: int) -> np.ndarray:
        out = np.empty(n, dtype=np.uint32)
        self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_challenger_sample(self.gpu.h, self.h, out.ctypes.data, n))
        return out

    def sample(self) -> int: return int(self.sample_many(1)[0])
    def sample_algebra_element(self) -> np.ndarray: return self.sample_many(4)

    def sample_bits(self, bits: int) -> int:
        """CanSampleBits: the duplex transcript masks the canonical value of one sample (duplex_challenger.rs:270-283), a byte
        transcript the raw u32 of 4 popped bytes.  2^bits must be below the field order (P3GpuError EINVAL otherwise)."""
        out = np.empty(1, dtype=np.uint32)
        self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_challenger_sample_bits(self.gpu.h, self.h, bits, 1, out.ctypes.data))
        return int(out[0])

    # ---- GrindingChallenger
    def grind(self, bits: int) -> int:
        w = C.c_uint32()
        self.gpu._use_torch_stream()
        check(self.gpu.L.p3gpu_challenger_grind(self.gpu.h, self.h, bits, C.byref(w)))
        return int(w.value)


def _host_words(values) -> np.ndarray:
    return np.ascontiguousarray(values.cpu().numpy().view(np.uint32) if _is_torch(values) else values, dtype=np.uint32).ravel()


class DuplexChallenger(_DeviceChallenger):
    """DuplexChallenger<F, Poseidon2<width>, width, rate>: examples use (Perm24, 24, 16) (examples/src/types.rs:56-60)."""

    def __init__(self, field: Field, perm: Poseidon2, rate: int, gpu):
        assert perm.field is field or perm.field == field
        self.field, self.perm, self.rate, self.gpu = field, perm, rate, gpu
        perm.upload(gpu)
        self._create(lambda out: gpu.L.p3gpu_challenger_new(gpu.h, field.id, perm.width, rate, out))


class SerializingChallenger32(_DeviceChallenger):
    """SerializingChallenger32<F, HashChallenger<u8, H, 32>> (challenger/src/serializing_challenger.rs, hash_challenger.rs) with
    H = Keccak256Hash, the transcript of the Keccak configuration (examples/src/types.rs:19-35), or H = Sha256, the transcript of
    the SHA-256 configurations (keccak-air/examples/prove_baby_bear_sha256*.rs); `hasher` is "keccak256" (the default) or
    "sha256".  Field elements are observed as the 4 little-endian bytes of their canonical values; a digest (8 words: [u64; 4] or
    [u8; 32]) as its 32 bytes; samples are rejection-sampled from 4 bytes popped off the end of the hash's digest; `sample_bits`
    masks the raw u32; `grind` returns the smallest witness."""

    HASHERS = ("keccak256", "sha256")

    def __init__(self, field: Field, gpu, hasher: str = "keccak256"):
        if hasher not in self.HASHERS:
            raise ValueError(f"unknown transcript hash {hasher!r} (one of {', '.join(self.HASHERS)})")
        self.field, self.gpu, self.hasher = field, gpu, hasher
        new = gpu.L.p3gpu_challenger_new_sha256 if hasher == "sha256" else gpu.L.p3gpu_challenger_new_keccak256
        self._create(lambda out: new(gpu.h, field.id, out))

    @classmethod
    def from_hasher(cls, initial_state, field: Field, gpu, hasher: str = "keccak256"):
        """from_hasher(initial_state, H): `initial_state` bytes become the start of the input buffer.  The transcript takes whole
        32-bit words, so their number must be a multiple of 4."""
        init = bytes(initial_state)
        if len(init) % 4:
            raise ValueError("the initial state must be a whole number of 32-bit words")
        c = cls(field, gpu, hasher)
        if init:
            c.observe_cap(np.frombuffer(init, dtype="<u4").astype(np.uint32))
        return c
