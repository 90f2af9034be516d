"""plonky3_b200 — H100-native backend for Plonky3's prover hot path (NTT/LDE -> Merkle -> FRI).

The compute lives in libp3gpu.so (plonky3_b200/csrc, C ABI in include/p3gpu.h); this package is the host-side mirror
of the reference's trait surfaces (TwoAdicSubgroupDft, Mmcs, FriParameters/FriFoldingStrategy, Pcs::commit).
There is no CPU fallback: without the built library and a CUDA device every entry point raises."""
from . import _lib
from ._lib import P3GpuError, HASH_KECCAK, HASH_POSEIDON2_W16, HASH_POSEIDON2_W24, HASH_SHA256, HASH_SHA256_COMPRESS
from .field import BabyBear, KoalaBear, Field, FIELDS

__all__ = ["_lib", "P3GpuError", "BabyBear", "KoalaBear", "Field", "FIELDS", "HASH_KECCAK", "HASH_POSEIDON2_W16",
           "HASH_POSEIDON2_W24", "HASH_SHA256", "HASH_SHA256_COMPRESS"]
