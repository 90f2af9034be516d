"""The SHA-256 configurations without a GPU: SHA-256 from the device source on the host against hashlib and the reference's own
vectors, the restated SHA-256 transcript (challenger/src/serializing_challenger.rs, hash_challenger.rs), the [u8; 32] wire form,
and the prove driver on the oracle-backed stand-in device answering the SHA-256 hash kinds with hashlib, verified by the product's
verifier."""
import hashlib
import json
import os
import pathlib
import subprocess

import numpy as np
import pytest
import torch

import sha256_air_oracle as SO
import sha256_config as S
from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4, DIGEST_U8X32, proof_from_postcard, proof_to_postcard

ROOT = pathlib.Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def sha256_host(tmp_path_factory):
    exe = tmp_path_factory.mktemp("sha256") / "sha256_host"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "sha256_host.cpp"), "-o", str(exe)],
                   check=True)

    def run(lines):
        r = subprocess.run([str(exe)], input="".join(l + "\n" for l in lines), capture_output=True, text=True, check=True)
        return r.stdout.split()
    return run


def test_device_sha256_published_vectors(sha256_host):
    got = sha256_host(["-", b"abc".hex(), b"hello world".hex()])
    assert got[0] == "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"
    assert got[1] == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"
    assert got[2] == "b94d27b9934d3e08a52e52d7da7dabfac484efe37a5380ee9088f7ace2efcde9"     # sha256/src/lib.rs test_hello_world


def test_device_sha256_matches_hashlib(sha256_host):
    rng = np.random.default_rng(9)
    msgs = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (0, 1, 55, 56, 63, 64, 65, 119, 120, 10532, 36672)]
    assert sha256_host([m.hex() or "-" for m in msgs]) == [hashlib.sha256(m).hexdigest() for m in msgs]


def test_device_compression_is_the_reference_sha256_compress(sha256_host):
    """sha256/src/lib.rs test_compress: compress([0; 32] || padding) from the IV is sha256([0; 32]); and random states and blocks
    agree with tests/sha256_air_oracle.compress."""
    iv = "".join("%08x" % v for v in SO.IV)
    pad = bytearray(32); pad[0] = 0x80; pad[30] = 1
    assert sha256_host([f"c {iv} {(bytes(32) + bytes(pad)).hex()}"])[0] == hashlib.sha256(bytes(32)).hexdigest()
    rng = np.random.default_rng(4)
    h = rng.integers(0, 1 << 32, (6, 8), dtype=np.uint32)
    blk = rng.integers(0, 1 << 32, (6, 16), dtype=np.uint32)
    want = SO.compress(h, blk)
    got = sha256_host([f"c {''.join('%08x' % v for v in h[i])} {''.join('%08x' % v for v in blk[i])}" for i in range(6)])
    assert got == ["".join("%08x" % v for v in want[i]) for i in range(6)]


def test_restated_mmcs_matches_the_reference_constructions():
    """The host Merkle restatement: a leaf is SHA-256 of the row's Montgomery words little-endian, the "hasher" node SHA-256 of the
    two digests' 64 bytes, the "compress" node one raw compression with big-endian output."""
    rows = np.array([[1, 2, 3], [0xFFFFFFFF, 0, 7]], dtype=np.uint32)
    assert S.hash_rows(rows)[1].astype("<u4").tobytes() == hashlib.sha256(rows[1].astype("<u4").tobytes()).digest()
    l, r = S.hash_rows(rows)
    assert S.compress_pairs([l], [r], "hasher")[0].astype("<u4").tobytes() == hashlib.sha256(l.astype("<u4").tobytes() + r.astype("<u4").tobytes()).digest()
    pad = bytearray(32); pad[0] = 0x80; pad[30] = 1
    zero, padw = np.zeros(8, dtype=np.uint32), np.frombuffer(bytes(pad), dtype="<u4")
    assert S.compress_pairs([zero], [padw], "compress")[0].astype("<u4").tobytes() == hashlib.sha256(bytes(32)).digest()


def test_abi_constants():
    assert (_lib.HASH_SHA256, _lib.HASH_SHA256_COMPRESS) == (3, 4)
    import plonky3_b200
    assert plonky3_b200.HASH_SHA256 == 3 and plonky3_b200.HASH_SHA256_COMPRESS == 4
    h = (ROOT / "include" / "p3gpu.h").read_text()
    rs = (ROOT / "bindings" / "rust" / "p3-gpu" / "src" / "ffi.rs").read_text()
    assert "P3GPU_HASH_SHA256 = 3," in h and "P3GPU_HASH_SHA256_COMPRESS = 4" in h
    assert "pub const P3GPU_HASH_SHA256: i32 = 3;" in rs and "pub const P3GPU_HASH_SHA256_COMPRESS: i32 = 4;" in rs
    assert "p3gpu_challenger_new_sha256" in h and "pub fn p3gpu_challenger_new_sha256(" in rs
    assert "p3gpu_challenger_new_sha256" in _lib.EXPORTS


# ---------------------------------------------------------------- the restated transcript
def test_samples_pop_from_the_end_of_the_digest():
    ch = S.transcript(BabyBear, bytes([0, 1, 2, 3]))
    d = hashlib.sha256(bytes([0, 1, 2, 3])).digest()
    assert ch.sample_bits(30) == int.from_bytes(d[28:32][::-1], "little") & ((1 << 30) - 1)
    assert ch.inner.input == bytearray(d)                         # the digest is the new input buffer
    assert ch.sample_bits(8) == d[27]                             # the next pop: bytes 27, 26, 25, 24
    ch.observe_canonical(5)
    assert ch.inner.output == bytearray() and bytes(ch.inner.input) == d + bytes([5, 0, 0, 0])
    d2 = hashlib.sha256(d + bytes([5, 0, 0, 0])).digest()
    assert ch.sample_bits(16) == int.from_bytes(d2[30:32][::-1], "little")


def test_field_samples_are_rejection_sampled():
    """A sample is the popped u32 with bit 31 dropped, redrawn while >= p."""
    ch = S.transcript(KoalaBear)
    d = hashlib.sha256(b"").digest()
    vals = [int.from_bytes(d[4 * k:4 * k + 4], "big") & 0x7FFFFFFF for k in range(7, -1, -1)]
    want = [v for v in vals if v < KoalaBear.P][:3]
    assert [KoalaBear.from_monty(int(v)) for v in ch.sample_many(3)] == want


def test_restated_grind_finds_the_smallest_witness():
    ch = S.transcript(BabyBear)
    ch.observe_slice(np.arange(1, 40, dtype=np.uint32))
    for bits in (1, 3, 6):
        before = ch.clone()
        w = ch.grind(bits)
        assert before.clone().check_witness(bits, w)
        assert not any(before.clone().check_witness(bits, BabyBear.to_monty(x)) for x in range(BabyBear.from_monty(w)))
        after = before.clone()
        after.check_witness(bits, w)                              # grind observes the witness and consumes the checked sample
        assert ch.inner.input == after.inner.input and ch.inner.output == after.inner.output


def test_zero_bit_grind_leaves_the_state_unchanged():
    ch = S.transcript(KoalaBear, bytes(8))
    shadow = ch.clone()
    assert ch.grind(0) == 0
    assert ch.inner.input == shadow.inner.input and ch.sample() == shadow.sample()


# ---------------------------------------------------------------- the [u8; 32] wire form
def _random_proof(rng):
    from types import SimpleNamespace
    d = lambda n: rng.integers(0, 1 << 32, (n, 8), dtype=np.uint32)
    e = lambda n: rng.integers(0, BabyBear.P, (n, 4), dtype=np.uint32)
    idx = [3, 9, 3]
    paths = rng.integers(0, 1 << 32, (3, 5, 8), dtype=np.uint32)
    return SimpleNamespace(trace_commit=d(8), quotient_commit=d(8), trace_local=e(6), trace_next=e(6), preprocessed_local=None,
                           preprocessed_next=None, quotient_chunks=[e(4), e(4)], commit_phase_commits=[d(8), d(4)],
                           commit_pow_witnesses=[0, 0], input_openings=[([rng.integers(0, BabyBear.P, (3, 5), dtype=np.uint32)], paths)],
                           input_opening_indices=[idx], commit_phase_openings=[(2, e(9).reshape(3, 3, 4), paths)],
                           commit_phase_indices=[idx], final_poly=e(1), query_pow_witness=777, degree_bits=9)


def test_u8x32_wire_round_trip_is_exact():
    from plonky3_b200.merkle_tree import prune_paths
    p = _random_proof(np.random.default_rng(5))
    raw = proof_to_postcard(p, DIGEST_U8X32)
    back = proof_from_postcard(raw, BabyBear.P, digest=DIGEST_U8X32)
    assert np.array_equal(back["trace_commit"], p.trace_commit) and np.array_equal(back["quotient_commit"], p.quotient_commit)
    assert all(np.array_equal(a, b) for a, b in zip(back["commit_phase_commits"], p.commit_phase_commits))
    assert np.array_equal(back["input_openings"][0]["proof"], prune_paths(p.input_opening_indices[0], p.input_openings[0][1]))
    assert np.array_equal(back["commit_phase_openings"][0]["proof"], prune_paths(p.commit_phase_indices[0], p.commit_phase_openings[0][2]))
    assert np.array_equal(back["trace_next"], p.trace_next) and back["query_pow_witness"] == 777 and back["degree_bits"] == 9
    # a cap is the Vec's varint length, then 32 raw bytes per digest: the words' little-endian bytes
    assert raw[0] == 8 and raw[1:1 + 256] == p.trace_commit.astype("<u4").tobytes() and raw[257] == 8
    assert proof_to_postcard(p, DIGEST_U8X32) == raw


def test_u8x32_reader_rejects_every_truncation():
    raw = proof_to_postcard(_random_proof(np.random.default_rng(6)), DIGEST_U8X32)
    for cut in range(len(raw)):
        with pytest.raises(ValueError):
            proof_from_postcard(raw[:cut], BabyBear.P, digest=DIGEST_U8X32)
    with pytest.raises(ValueError, match="trailing"):
        proof_from_postcard(raw + b"\x00", BabyBear.P, digest=DIGEST_U8X32)
    with pytest.raises(ValueError, match="codec"):
        proof_from_postcard(raw, BabyBear.P, digest="u8x16")


def test_other_codecs_bytes_unchanged():
    """The reference's [F; 8] fixture still reads and re-encodes byte for byte; a [u64; 4] proof is still varint lanes; digests
    whose words all lie below p are the same bytes under f8 and u8x32."""
    from plonky3_b200.proof_io import _vec_of_digests
    gold = json.loads((ROOT / "tests" / "golden" / "uni_stark_two_adic_v1.json").read_text())
    raw = bytes.fromhex(gold["postcard_hex"])
    d = proof_from_postcard(raw, BabyBear.P)
    assert raw.startswith(_vec_of_digests(d["trace_commit"], DIGEST_F8) + _vec_of_digests(d["quotient_commit"], DIGEST_F8))
    a = np.array([[1, 0, 2, 0, 3, 0, 4, 0]], dtype=np.uint32)
    assert _vec_of_digests(a, DIGEST_U64X4) == bytes([1, 1, 2, 3, 4])
    assert _vec_of_digests(a, DIGEST_F8) == _vec_of_digests(a, DIGEST_U8X32) == bytes([1]) + a.astype("<u4").tobytes()


# ---------------------------------------------------------------- the prove driver on the stand-in device
@pytest.fixture
def no_sync(monkeypatch):
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)      # the driver's span timers synchronise the device


@pytest.mark.parametrize("node", ["hasher", "compress"])
def test_prove_driver_on_the_stand_in_device(no_sync, node):
    """uni_stark.prove with Sha256StarkConfig's shape on the stand-in device (the SHA-256 hash kinds answered by hashlib, the
    transcript restated); the product verifier with the hashlib MMCS accepts the wire proof and rejects corruptions."""
    import air_examples as E
    from plonky3_b200.air import SymbolicAir
    from plonky3_b200.uni_stark import prove
    from plonky3_b200.verifier import VerificationError, verify
    f, n = BabyBear, 1 << 5
    fri = (1, 0, 2, 6, 0, 3)
    from test_air_preprocessed_cpu import LayoutMockGpu
    mock = S.with_sha256(LayoutMockGpu)()
    config = S.mock_config(f, mock, node, fri, 1)
    trace = E.fib_trace(f, n)
    pis = [0, 1, f.from_monty(int(trace[-1, 1]))]
    air = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=mock)
    proof = prove(config, air, torch.from_numpy(trace.view(np.int32)), pis)
    assert proof.digest_codec == DIGEST_U8X32
    raw = proof.to_postcard()
    vcfg = S.verifier_config(f, node, fri)
    verify(vcfg, air, raw, pis)
    with pytest.raises(VerificationError):
        verify(vcfg, air, raw, pis[:2] + [pis[2] + 1])
    with pytest.raises(VerificationError):                          # the other node compression does not verify it
        verify(S.verifier_config(f, "compress" if node == "hasher" else "hasher", fri), air, raw, pis)
    for pos in (5, 1 + 32 * len(proof.trace_commit) + 3, len(raw) - 6):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, air, bytes(bad), pis)
