"""The byte transcript's state machine without a GPU: the functions of plonky3_b200/csrc/hash_core.cuh that the challenger kernels
run (observe, flush, pop, sample, the grind's witness test from the midstate), compiled with g++ and driven through
tests/cpp/transcript_host.cpp.  The scripts are those of the GPU transcript tests (test_gpu_prove_keccak.py,
test_gpu_sha256_config.py): random observe / sample / clone sequences and grinds after pending tails that end on every block
boundary case, compared with the restatements tests/keccak_transcript.SerializingChallenger32 (Keccak-256) and
tests/sha256_config.transcript (SHA-256)."""
import os
import pathlib
import subprocess

import numpy as np
import pytest

import keccak_transcript as K
import sha256_config as S
from plonky3_b200.field import BabyBear, KoalaBear

ROOT = pathlib.Path(__file__).resolve().parent.parent
FIELDS = pytest.mark.parametrize("field", [BabyBear, KoalaBear], ids=["bb", "kb"])


class Filter:
    """One running transcript_host: a command line in, its one answer line out."""

    def __init__(self, exe):
        self.p = subprocess.Popen([str(exe)], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, line: str) -> str:
        self.p.stdin.write(line + "\n")
        self.p.stdin.flush()
        out = self.p.stdout.readline()
        assert out, f"transcript_host stopped at {line!r} (exit {self.p.poll()})"
        return out.strip()

    def close(self):
        self.p.stdin.close()
        assert self.p.wait(timeout=60) == 0


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    exe = tmp_path_factory.mktemp("transcript") / "transcript_host"
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-w", "-I", cuda_inc, str(ROOT / "tests" / "cpp" / "transcript_host.cpp"),
                    "-o", str(exe)], check=True)
    f = Filter(exe)
    yield f
    f.close()


def _line(words) -> str:
    return " ".join(str(int(w)) for w in np.asarray(words, dtype=np.uint32).ravel())


class HostTranscript:
    """The surface of plonky3_b200.challenger.SerializingChallenger32 on one transcript of the filter."""

    def __init__(self, host, field, handle):
        self.host, self.field, self.handle = host, field, handle

    @classmethod
    def from_hasher(cls, host, initial_state, field, hasher):
        init = np.frombuffer(bytes(initial_state), dtype="<u4")
        return cls(host, field, host.ask(f"new {hasher[0]} {field.id} {_line(init)}"))

    def _ask(self, cmd: str) -> str: return self.host.ask(f"{self.handle} {cmd}")
    def clone(self): return HostTranscript(self.host, self.field, self._ask("clone"))
    def observe_slice(self, values): assert self._ask(f"obs {_line(values)}") == "ok"
    def observe(self, value: int): self.observe_slice([value])
    def observe_canonical(self, x: int): self.observe(self.field.to_monty(x))
    def observe_cap(self, cap): assert self._ask(f"dig {_line(cap)}") == "ok"
    def sample_many(self, n: int) -> np.ndarray: return np.array(self._ask(f"sample {n}").split(), dtype=np.uint32)
    def sample(self) -> int: return int(self.sample_many(1)[0])
    def sample_algebra_element(self) -> np.ndarray: return self.sample_many(4)
    def sample_bits(self, bits: int) -> int: return int(self._ask(f"bits {bits}"))
    def grind(self, bits: int) -> int: return 0 if bits == 0 else int(self._ask(f"grind {bits}"))


def _restated(hasher, field, initial_state=b""):
    return S.transcript(field, initial_state) if hasher == "sha256" else K.SerializingChallenger32.from_hasher(field, initial_state)


def _script(rng, pairs, field, steps, max_host, max_dev):
    """The GPU tests' random script; "device-resident" observes are plain observes here, kept so the draws match."""
    for step in range(steps):
        d, r = pairs[rng.integers(0, len(pairs))]
        op = rng.integers(0, 7)
        if op == 0:
            v = rng.integers(0, field.P, int(rng.integers(0, max_host)), dtype=np.uint32)
            d.observe_slice(v); r.observe_slice(v)
        elif op == 1:
            v = rng.integers(0, field.P, int(rng.integers(1, max_dev)), dtype=np.uint32)
            d.observe_slice(v); r.observe_slice(v)
        elif op == 2:                                              # a cap of digests: any 32-bit words
            v = rng.integers(0, 1 << 32, (1 << int(rng.integers(0, 4)), 8), dtype=np.uint32)
            d.observe_cap(v); r.observe_cap(v)
        elif op == 3:
            n = int(rng.integers(1, 12))
            assert list(d.sample_many(n)) == list(r.sample_many(n))
        elif op == 4:
            bits = int(rng.integers(0, 31))
            assert d.sample_bits(bits) == r.sample_bits(bits)
        elif op == 5:
            x = int(rng.integers(0, 1000))
            d.observe_canonical(x); r.observe_canonical(x)
        elif len(pairs) < 4:
            pairs.append((d.clone(), r.clone()))
    for d, r in pairs:                                             # every clone ran its own transcript
        assert list(d.sample_algebra_element()) == list(r.sample_algebra_element())


@FIELDS
def test_keccak256_transcript_matches_restatement(host, field):
    rng = np.random.default_rng(17 + field.id)
    pairs = [(HostTranscript.from_hasher(host, b"", field, "keccak256"), _restated("keccak256", field))]
    _script(rng, pairs, field, 120, 80, 300)


@FIELDS
def test_sha256_transcript_matches_restatement(host, field):
    rng = np.random.default_rng(23 + field.id)
    init = rng.integers(0, 256, 12, dtype=np.uint8).tobytes()
    pairs = [(HostTranscript.from_hasher(host, init, field, "sha256"), _restated("sha256", field, init))]
    _script(rng, pairs, field, 150, 40, 200)
    fresh = HostTranscript.from_hasher(host, b"", field, "sha256")
    assert list(fresh.sample_many(3)) == list(_restated("sha256", field).sample_many(3))


@FIELDS
def test_keccak256_grind_is_the_sequential_smallest_witness(host, field):
    """Pending tails of 0, 0 after a full block, 33 (the candidate completes the block, the padding needs a second one) and 20
    words; some after a flush, where the digest is the pending input."""
    rng = np.random.default_rng(5)
    for bits in range(1, 17):
        ch, rs = HostTranscript.from_hasher(host, b"", field, "keccak256"), _restated("keccak256", field)
        prefix = [0, 34, 33, 34 * 3 + 20][bits % 4]
        v = rng.integers(0, field.P, prefix, dtype=np.uint32)
        ch.observe_slice(v); rs.observe_slice(v)
        if bits % 5 == 0:
            assert ch.sample() == rs.sample()
        assert ch.grind(bits) == rs.grind(bits), bits
        assert list(ch.sample_many(2)) == list(rs.sample_many(2))
    ch, rs = HostTranscript.from_hasher(host, b"", field, "keccak256"), _restated("keccak256", field)
    v = rng.integers(0, field.P, 57, dtype=np.uint32)
    ch.observe_slice(v); rs.observe_slice(v)
    w = ch.grind(20)
    assert rs.clone().check_witness(20, w)
    assert rs.check_witness(20, w) and list(ch.sample_many(4)) == list(rs.sample_many(4))


@FIELDS
def test_sha256_grind_is_the_sequential_smallest_witness(host, field):
    """Pending tails of 0, 13 (the length no longer fits: two blocks), 15 (the candidate completes the block) and 13 words beyond
    full blocks; some after a flush, where the digest is the pending input."""
    rng = np.random.default_rng(31)
    for bits in range(1, 13):
        ch, rs = HostTranscript.from_hasher(host, b"", field, "sha256"), _restated("sha256", field)
        prefix = [0, 13, 15, 16 * 2 + 13][bits % 4]
        v = rng.integers(0, field.P, prefix, dtype=np.uint32)
        ch.observe_slice(v); rs.observe_slice(v)
        if bits % 3 == 0:
            assert ch.sample() == rs.sample()
        assert ch.grind(bits) == rs.grind(bits), bits
        assert list(ch.sample_many(2)) == list(rs.sample_many(2))


@pytest.mark.parametrize("hasher", ["keccak256", "sha256"])
def test_witness_test_is_check_witness(host, hasher):
    """The grind kernel's per-candidate test, which finishes the hash from the midstate, against observe + sample_bits on a clone,
    for candidates around every pending length of a block."""
    field = KoalaBear
    rng = np.random.default_rng(11)
    ch, rs = HostTranscript.from_hasher(host, b"", field, hasher), _restated(hasher, field)
    for _ in range(40):
        bits = int(rng.integers(1, 5))
        for c in rng.integers(0, field.P, 4):
            want = rs.clone().check_witness(bits, field.to_monty(int(c)))
            assert ch._ask(f"wit {bits} {int(c)}") == str(int(want))
        v = rng.integers(0, field.P, 1, dtype=np.uint32)
        ch.observe_slice(v); rs.observe_slice(v)
