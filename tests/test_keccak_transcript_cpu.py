"""The Keccak configuration without a GPU: Keccak-256 from the device source on the host, the restated transcript's plumbing
(challenger/src/serializing_challenger.rs and hash_challenger.rs, including what the reference's own ByteCountHasher tests pin), the
[u64; 4] wire form, and the prove driver on the oracle-backed stand-in device, verified by the product's verifier."""
import json
import os
import pathlib
import subprocess

import numpy as np
import pytest
import torch

import keccak_transcript as K
from oracle import p3_oracle as O
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.proof_io import DIGEST_U64X4, proof_from_postcard, proof_to_postcard

ROOT = pathlib.Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def keccak256_host(tmp_path_factory):
    exe = tmp_path_factory.mktemp("k256") / "keccak256_host"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "keccak256_host.cpp"), "-o", str(exe)],
                   check=True)

    def run(msgs):
        text = "".join((m.hex() or "-") + "\n" for m in msgs)
        r = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True)
        return [bytes.fromhex(x) for x in r.stdout.split()]
    return run


def test_device_keccak256_published_vectors(keccak256_host):
    got = keccak256_host([b"", b"abc"])
    assert got[0].hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert got[1].hex() == "4e03657aea45a94fc7d47ba826c8d667c0d1e6e33a64a036ec44f58fa12d6c45"
    assert K.keccak256(b"").hex().startswith("c5d24601") and K.keccak256(b"abc").hex().endswith("a12d6c45")


def test_device_keccak256_matches_restatement(keccak256_host):
    rng = np.random.default_rng(7)
    msgs = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (0, 1, 4, 135, 136, 137, 271, 272, 273, 21000, 21011)]
    assert keccak256_host(msgs) == [K.keccak256(m) for m in msgs]


def _byte_count(msg: bytes) -> bytes:
    """ByteCountHasher (serializing_challenger.rs tests): byte i of the digest = len + i (mod 256)."""
    return bytes((len(msg) + i) & 0xFF for i in range(32))


def _bc(field=BabyBear):
    return K.SerializingChallenger32.from_hasher(field, bytes([0, 1, 2, 3]), _byte_count)


def test_zero_bit_grind_leaves_the_state_unchanged():
    ch = _bc()
    shadow = ch.clone()
    assert ch.grind(0) == 0
    assert ch.inner.sample_byte() == shadow.inner.sample_byte()
    assert ch.inner.input == shadow.inner.input


@pytest.mark.parametrize("field", [BabyBear, KoalaBear])
def test_oversized_bit_counts_are_rejected(field):
    with pytest.raises(AssertionError, match="field order"):
        _bc(field).sample_bits(32)
    with pytest.raises(AssertionError, match="field order"):
        _bc(field).grind(32)
    with pytest.raises(AssertionError, match="field order"):
        _bc(field).sample_bits(31)                               # 2^31 > p for both fields
    _bc(field).sample_bits(30)


def test_samples_pop_from_the_end_of_the_digest():
    ch = _bc()
    # 4 bytes observed: the flush hashes 4 bytes -> digest bytes 4, 5, ..., 35; popped last-first: 35, 34, 33, 32
    assert ch.sample_bits(30) == int.from_bytes(bytes([35, 34, 33, 32]), "little") & ((1 << 30) - 1)
    assert ch.inner.input == bytearray(range(4, 36))             # the digest is the new input buffer
    assert ch.sample_bits(8) == 31                               # next pop: bytes 31, 30, 29, 28 -> low byte 31
    ch.observe_canonical(5)                                      # clears the output; the input is digest || 05 00 00 00
    assert ch.inner.output == bytearray() and len(ch.inner.input) == 36
    assert ch.sample_bits(8) == (36 + 31) & 0xFF                 # the re-absorbed digest counts: 36 bytes hashed


def test_field_samples_are_rejection_sampled():
    # digest bytes all 0xff: u32 = 0xffffffff -> 0x7fffffff >= p (rejected) until the output buffer runs dry and is refilled
    def hasher(msg):
        return bytes([0xFF] * 32) if len(msg) != 32 else bytes(range(32))
    ch = K.SerializingChallenger32.from_hasher(BabyBear, b"", hasher)
    v = ch.sample()
    assert BabyBear.from_monty(v) == int.from_bytes(bytes([31, 30, 29, 28]), "little") & 0x7FFFFFFF
    # a value below p after masking is kept: bit 31 is dropped, not reduced
    ch2 = K.SerializingChallenger32.from_hasher(BabyBear, b"", lambda m: bytes([1, 0, 0, 0x80] * 8))
    assert BabyBear.from_monty(ch2.sample()) == int.from_bytes(bytes([0x80, 0, 0, 1]), "little") & 0x7FFFFFFF


def test_restated_grind_finds_the_smallest_witness():
    ch = K.SerializingChallenger32.from_hasher(KoalaBear)
    ch.observe_slice(np.arange(1, 200, dtype=np.uint32))
    for bits in (1, 4, 9):
        lit = ch.clone()
        lit.inner.hasher = lambda m: K.keccak256(m)              # not `keccak256` itself: the literal per-candidate path
        before = lit.clone()
        w = ch.grind(bits)
        assert lit.grind(bits) == w
        assert ch.inner.input == lit.inner.input and ch.inner.output == lit.inner.output
        assert before.clone().check_witness(bits, w)
        assert not any(before.clone().check_witness(bits, KoalaBear.to_monty(x)) for x in range(KoalaBear.from_monty(w)))


def _random_digest_proof(rng, codec_lanes_big: bool):
    from types import SimpleNamespace
    d = lambda n: rng.integers(0, 1 << 32, (n, 8), dtype=np.uint32) if codec_lanes_big else rng.integers(0, 200, (n, 8), dtype=np.uint32)
    e = lambda n: rng.integers(0, KoalaBear.P, (n, 4), dtype=np.uint32)
    idx = [3, 9, 3]
    paths = rng.integers(0, 1 << 32, (3, 5, 8), dtype=np.uint32)
    return SimpleNamespace(trace_commit=d(8), quotient_commit=d(8), trace_local=e(6), trace_next=None, preprocessed_local=e(2),
                           preprocessed_next=None, quotient_chunks=[e(4), e(4)], commit_phase_commits=[d(8), d(4)],
                           commit_pow_witnesses=[0, 0], input_openings=[([rng.integers(0, KoalaBear.P, (3, 5), dtype=np.uint32)], paths)],
                           input_opening_indices=[idx], commit_phase_openings=[(2, e(9).reshape(3, 3, 4), paths)],
                           commit_phase_indices=[idx], final_poly=e(1), query_pow_witness=12345, degree_bits=7)


@pytest.mark.parametrize("big", [True, False])
def test_u64x4_wire_round_trip_is_exact(big):
    from plonky3_b200.merkle_tree import prune_paths
    p = _random_digest_proof(np.random.default_rng(3 + big), big)
    raw = proof_to_postcard(p, DIGEST_U64X4)
    back = proof_from_postcard(raw, KoalaBear.P, digest=DIGEST_U64X4)
    assert np.array_equal(back["trace_commit"], p.trace_commit) and np.array_equal(back["quotient_commit"], p.quotient_commit)
    assert all(np.array_equal(a, b) for a, b in zip(back["commit_phase_commits"], p.commit_phase_commits))
    assert np.array_equal(back["input_openings"][0]["proof"], prune_paths(p.input_opening_indices[0], p.input_openings[0][1]))
    assert np.array_equal(back["commit_phase_openings"][0]["proof"], prune_paths(p.commit_phase_indices[0], p.commit_phase_openings[0][2]))
    assert np.array_equal(back["preprocessed_local"], p.preprocessed_local) and back["query_pow_witness"] == 12345
    # every u64 is a varint: the cap alone is 1 + sum of the lanes' varint lengths
    lanes = p.trace_commit.astype(np.uint64)[:, 0::2] | (p.trace_commit.astype(np.uint64)[:, 1::2] << np.uint64(32))
    assert raw[0] == 8 and raw[1 + sum(max(1, (int(v).bit_length() + 6) // 7) for v in lanes.ravel())] == 8
    assert proof_to_postcard(p, DIGEST_U64X4) == raw
    # writing the parsed dict's digests back gives the same bytes (the [F; 8] default would not)
    assert proof_to_postcard(p) != raw


def test_u64x4_reader_rejects_malformed_input():
    p = _random_digest_proof(np.random.default_rng(11), True)
    raw = proof_to_postcard(p, DIGEST_U64X4)
    for cut in (1, 5, 40, len(raw) // 2, len(raw) - 1):
        with pytest.raises(ValueError):
            proof_from_postcard(raw[:cut], KoalaBear.P, digest=DIGEST_U64X4)
    with pytest.raises(ValueError, match="trailing"):
        proof_from_postcard(raw + b"\x00", KoalaBear.P, digest=DIGEST_U64X4)
    # an 11-byte varint for the first lane, and a 10-byte one whose value reaches 2^64
    overlong = bytes([1]) + bytes([0x80] * 10 + [0x00])
    with pytest.raises(ValueError, match="10 bytes"):
        proof_from_postcard(overlong + raw[1:], KoalaBear.P, digest=DIGEST_U64X4)
    too_big = bytes([1]) + bytes([0xFF] * 9 + [0x02])
    with pytest.raises(ValueError, match="range"):
        proof_from_postcard(too_big + raw[1:], KoalaBear.P, digest=DIGEST_U64X4)
    # the Option tags (random commitment, trace_next) flipped to 1 / 2
    d = proof_from_postcard(raw, KoalaBear.P, digest=DIGEST_U64X4)
    assert d["trace_next"] is None
    from plonky3_b200.proof_io import _vec_of_digests
    n_caps = len(_vec_of_digests(p.trace_commit, DIGEST_U64X4)) + len(_vec_of_digests(p.quotient_commit, DIGEST_U64X4))
    for pos, val in ((n_caps, 1), (n_caps, 2)):
        bad = bytearray(raw); bad[pos] = val
        with pytest.raises(ValueError):
            proof_from_postcard(bytes(bad), KoalaBear.P, digest=DIGEST_U64X4)
    with pytest.raises(ValueError, match="codec"):
        proof_from_postcard(raw, KoalaBear.P, digest="u64x8")


def test_default_codec_bytes_unchanged():
    """The reference's [F; 8] fixture (1115 bytes) reads the same through the default codec and the explicit one, and its digests
    re-encode to the fixture's own bytes."""
    from plonky3_b200.proof_io import DIGEST_F8, _vec_of_digests
    gold = json.loads((ROOT / "tests" / "golden" / "uni_stark_two_adic_v1.json").read_text())
    raw = bytes.fromhex(gold["postcard_hex"])
    assert len(raw) == 1115
    d, e = proof_from_postcard(raw, BabyBear.P), proof_from_postcard(raw, BabyBear.P, digest=DIGEST_F8)
    assert np.array_equal(d["trace_commit"], e["trace_commit"]) and d["degree_bits"] == e["degree_bits"]
    caps = _vec_of_digests(d["trace_commit"], DIGEST_F8) + _vec_of_digests(d["quotient_commit"], DIGEST_F8)
    assert raw.startswith(caps)
    for o in d["input_openings"] + d["commit_phase_openings"]:
        assert _vec_of_digests(o["proof"], DIGEST_F8) in raw
    with pytest.raises(ValueError):
        proof_from_postcard(raw, BabyBear.P, digest=DIGEST_U64X4)      # the other codec does not read it as a proof


@pytest.fixture
def no_sync(monkeypatch):
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)      # the driver's span timers synchronise the device


@pytest.mark.parametrize("log_rows,num_queries,pow_bits", [(3, 4, 3), (5, 9, 6)])
def test_keccak_prove_driver_on_the_stand_in_device(no_sync, log_rows, num_queries, pow_bits):
    """uni_stark.prove with the Keccak configuration's shape — every transcript call through the restated
    SerializingChallenger32 — on the oracle-backed stand-in device; the product verifier (oracle Keccak MMCS hashing, restated
    transcript) accepts the wire proof and rejects corrupted caps, sibling hashes, witnesses and opened values."""
    from plonky3_b200.verifier import VerificationError, verify
    proof, air = K.mock_prove_p2(KoalaBear, log_rows, num_queries, pow_bits)
    assert proof.digest_codec == DIGEST_U64X4
    raw = proof.to_postcard()
    vcfg = K.verifier_config(KoalaBear, num_queries, pow_bits)
    verify(vcfg, air, raw)
    # the query proof-of-work witness: the restatement's smallest
    assert proof.query_pow_witness == KoalaBear.to_monty(KoalaBear.from_monty(proof.query_pow_witness))
    for pos in _corruption_sites(raw, proof):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, air, bytes(bad))


def _corruption_sites(raw: bytes, proof) -> list:
    """Byte offsets inside: the trace cap, the first opened value, the first pruned sibling hash of the first input batch, and
    the query proof-of-work witness."""
    from plonky3_b200.proof_io import _vec_of_digests
    cap = len(_vec_of_digests(proof.trace_commit, DIGEST_U64X4))
    qcap = len(_vec_of_digests(proof.quotient_commit, DIGEST_U64X4))
    opened = cap + qcap + 1 + 2                                      # random tag, then Vec<EF> length (2 bytes for 1312 values)
    return [3, opened + 1, len(raw) - 6, raw.index(_vec_of_digests(_first_sibling(proof), DIGEST_U64X4)[1:]) + 1]


def _first_sibling(proof):
    from plonky3_b200.merkle_tree import prune_paths
    (rows, paths), idx = proof.input_openings[0], proof.input_opening_indices[0]
    return prune_paths(idx, paths)[:1]
