"""The SHA-256 configurations on the GPU (uni_stark.Sha256StarkConfig: a SHA-256 MMCS with either node compression, and
SerializingChallenger32 over SHA-256 resident on the device), against hashlib restatements (tests/sha256_config.py):

  - Merkle commits of both hash kinds over both fields, layer by layer: widths around the 16-word block, the Keccak AIR's 2633
    columns, non-power-of-two heights, several matrices of one height, injected shorter matrices, more than 8 matrices per
    height (the device table), cap heights 0 and 3; pcs_commit, fri_commit_phase and merkle_from_digests;
  - the device transcript against the restated one on random scripts, and its proof-of-work search;
  - the reference's two example statements (prove_baby_bear_sha256 / _sha256_compress: KeccakAir, 1,365 hashes, new_benchmark,
    cap height 3), and the same checks over KoalaBear, for the DSL Fibonacci AIR with public values and for an AIR with
    preprocessed and periodic columns: prove -> verify, the host verifier (hashlib MMCS, restated transcript) accepts the wire
    proof, a flipped byte in each section is rejected;
  - prove_sharded under Sha256StarkConfig writes prove's bytes (world 1, and 2 ranks sharing the card)."""
import hashlib
import os

import numpy as np
import pytest
import torch

import sha256_config as S
from plonky3_b200 import _lib
from plonky3_b200.challenger import SerializingChallenger32
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu, default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs, prune_paths
from plonky3_b200.proof_io import DIGEST_U8X32
from plonky3_b200.uni_stark import Sha256StarkConfig, prove, setup_preprocessed, verify
from plonky3_b200.verifier import VerificationError

pytestmark = pytest.mark.gpu
KINDS = {"hasher": _lib.HASH_SHA256, "compress": _lib.HASH_SHA256_COMPRESS}


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32) if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.uint32)


def rand(f, h, w, seed):
    return np.random.default_rng(seed).integers(0, f.P, (h, w), dtype=np.uint32)


# ---------------------------------------------------------------- Merkle commits
SHAPES = {
    "widths": [[(37, w)] for w in (1, 15, 16, 17, 100, 2633)],
    "one_height": [[(64, 3), (64, 16), (64, 5)]],
    "mixed_heights": [[(37, 17), (19, 5), (10, 100), (5, 1)], [(64, 8), (32, 40), (32, 1), (2, 3)]],
    "device_table": [[(24, w) for w in range(1, 11)] + [(12, w) for w in range(3, 15)]],
}


@pytest.mark.parametrize("node", sorted(KINDS))
@pytest.mark.parametrize("field", [BabyBear, KoalaBear], ids=["bb", "kb"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_merkle_commit_matches_hashlib(gpu, node, field, shape):
    for k, dims in enumerate(SHAPES[shape]):
        mats = [rand(field, h, w, 100 * k + i) for i, (h, w) in enumerate(dims)]
        want = S.merkle_tree(mats, node)
        layers = gpu.merkle_commit(field.id, KINDS[node], [dev(m) for m in mats])
        assert len(layers) == len(want)
        for l, (a, b) in enumerate(zip(layers, want)):
            assert np.array_equal(host(a), b), (dims, l)
        for cap_height in (0, 3):
            mmcs = MerkleTreeMmcs.sha256(field, cap_height=cap_height, gpu=gpu, node=node)
            cap, _ = mmcs.commit([dev(m) for m in mats])
            assert np.array_equal(host(cap), S.cap(want, cap_height))


def test_unknown_hash_kind_is_unsupported(gpu):
    m = dev(rand(BabyBear, 8, 4, 1))
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.merkle_commit(BabyBear.id, 5, [m])
    assert ex.value.code == _lib.EUNSUPPORTED
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.merkle_from_digests(BabyBear.id, 5, dev(np.zeros((4, 8), dtype=np.uint32)))
    assert ex.value.code == _lib.EUNSUPPORTED
    with pytest.raises(ValueError):
        MerkleTreeMmcs.sha256(BabyBear, node="sponge")


@pytest.mark.parametrize("node", sorted(KINDS))
def test_pcs_commit_fri_and_digest_layers(gpu, node):
    from oracle import p3_oracle as O
    f = KoalaBear
    m = rand(f, 1 << 8, 45, 3)
    lde, layers = gpu.pcs_commit(f.id, KINDS[node], dev(m), 1)
    assert np.array_equal(host(lde), O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True))
    want = S.merkle_tree([host(lde)], node)
    assert all(np.array_equal(host(a), b) for a, b in zip(layers, want)) and len(layers) == len(want)

    vec = rand(f, 1 << 10, 4, 5)
    betas = rand(f, 16, 4, 6)                                      # enough rounds for arity 2
    for max_log_arity, cap_height in ((3, 3), (1, 0)):
        caps, las, final = gpu.fri_commit_phase(f.id, KINDS[node], dev(vec), 1, 0, max_log_arity, cap_height, betas)
        wcaps, wlas, wfinal = S.fri_commit_phase(f.id, node, cap_height, vec, 1, 0, max_log_arity, betas)
        assert las == wlas and len(caps) == len(wcaps) and np.array_equal(final, wfinal)
        assert all(np.array_equal(a, b) for a, b in zip(caps, wcaps))

    digests = np.random.default_rng(8).integers(0, 1 << 32, (13, 8), dtype=np.uint32)
    got = gpu.merkle_from_digests(f.id, KINDS[node], dev(digests))
    cur = np.zeros((14, 8), dtype=np.uint32); cur[:13] = digests
    assert np.array_equal(host(got[0]), cur)
    for layer in got[1:]:
        raw = cur.shape[0] // 2
        nxt = np.zeros((raw if raw <= 1 else (raw + 1) // 2 * 2, 8), dtype=np.uint32)
        nxt[:raw] = S.compress_pairs(cur[0:2 * raw:2], cur[1:2 * raw:2], node)
        assert np.array_equal(host(layer), nxt)
        cur = nxt
    assert cur.shape[0] == 1


# ---------------------------------------------------------------- the transcript
@pytest.mark.parametrize("field", [BabyBear, KoalaBear], ids=["bb", "kb"])
def test_device_transcript_matches_restatement(gpu, field):
    rng = np.random.default_rng(23 + field.id)
    init = rng.integers(0, 256, 12, dtype=np.uint8).tobytes()
    ch = SerializingChallenger32.from_hasher(init, field, gpu, hasher="sha256")
    pairs = [(ch, S.transcript(field, init))]
    for step in range(150):
        d, r = pairs[rng.integers(0, len(pairs))]
        op = rng.integers(0, 7)
        if op == 0:                                                # host field elements, across block boundaries
            v = rng.integers(0, field.P, int(rng.integers(0, 40)), dtype=np.uint32)
            d.observe_slice(v); r.observe_slice(v)
        elif op == 1:                                              # device-resident field elements
            v = rng.integers(0, field.P, int(rng.integers(1, 200)), dtype=np.uint32)
            d.observe_slice(dev(v)); r.observe_slice(v)
        elif op == 2:                                              # a cap of [u8; 32] digests: any 32-bit words
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
    for d, r in pairs:
        assert list(d.sample_algebra_element()) == list(r.sample_algebra_element())
    fresh = SerializingChallenger32.from_hasher([], field, gpu, hasher="sha256")
    assert list(fresh.sample_many(3)) == list(S.transcript(field).sample_many(3))
    with pytest.raises(ValueError):
        SerializingChallenger32.from_hasher(b"abc", field, gpu, hasher="sha256")


def test_device_transcript_rejects_bad_input_before_launch(gpu):
    ch = SerializingChallenger32.from_hasher([], KoalaBear, gpu, hasher="sha256")
    n0 = gpu.launches
    for bits in (31, 32, 40):
        with pytest.raises(_lib.P3GpuError) as ex:
            ch.grind(bits)
        assert ex.value.code == _lib.EINVAL
        with pytest.raises(_lib.P3GpuError) as ex:
            ch.sample_bits(bits)
        assert ex.value.code == _lib.EINVAL
    assert gpu.launches == n0
    assert ch.grind(0) == 0 and gpu.launches == n0                 # 0 bits: no search, the state untouched
    assert list(ch.sample_many(3)) == list(S.transcript(KoalaBear).sample_many(3))


def _late_witness_prefix(field, bits):
    """A canonical value x such that after observe(x) no candidate of the first grind launch (2^(bits+3) of them) is a witness."""
    mask, batch = (1 << bits) - 1, 1 << (bits + 3)
    for x in range(1 << 22):
        pre = hashlib.sha256(x.to_bytes(4, "little"))
        if all(int.from_bytes(_fin(pre, c)[28:], "big") & mask for c in range(batch)):
            return x
    raise AssertionError("no prefix found")


def _fin(h, c):
    h = h.copy()
    h.update(c.to_bytes(4, "little"))
    return h.digest()


@pytest.mark.parametrize("field", [BabyBear, KoalaBear], ids=["bb", "kb"])
def test_grind_returns_the_sequential_smallest_witness(gpu, field):
    """Pending tails of 0, 13 (the length no longer fits: two blocks), 15 (the candidate completes the block) and 8 (after a flush)
    words, beyond full blocks; and a witness past the first launch batch."""
    rng = np.random.default_rng(31)
    for bits in range(1, 13):
        ch = SerializingChallenger32.from_hasher([], field, gpu, hasher="sha256")
        rs = S.transcript(field)
        prefix = [0, 13, 15, 16 * 2 + 13][bits % 4]
        v = rng.integers(0, field.P, prefix, dtype=np.uint32)
        ch.observe_slice(v); rs.observe_slice(v)
        if bits % 3 == 0:                                          # after a flush: the digest is the pending input
            assert ch.sample() == rs.sample()
        w = ch.grind(bits)
        assert w == rs.grind(bits), bits
        assert list(ch.sample_many(2)) == list(rs.sample_many(2))
    x = _late_witness_prefix(field, 1)
    ch, rs = SerializingChallenger32.from_hasher([], field, gpu, hasher="sha256"), S.transcript(field)
    ch.observe_canonical(x); rs.observe_canonical(x)
    w = ch.grind(1)
    assert field.from_monty(w) >= 16 and w == rs.grind(1)
    assert list(ch.sample_many(2)) == list(rs.sample_many(2))


# ---------------------------------------------------------------- proofs
def _config(gpu, field, node, fri, cap_height):
    m = MerkleTreeMmcs.sha256(field, cap_height=cap_height, gpu=gpu, node=node)
    return Sha256StarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m, FriParameters(*fri, m)))


def _sections(raw, proof):
    """A byte inside every section of the wire proof: both caps, the opened trace row, a quotient chunk, a FRI commit-phase cap,
    an opened input row and a pruned sibling hash of the first batch, a commit-phase sibling value and pruned sibling hash, the
    final polynomial, the query proof-of-work witness and degree_bits."""
    b = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.uint32)).astype("<u4").tobytes()
    (rows, paths), idx = proof.input_openings[0], proof.input_opening_indices[0]
    la, sib, cpaths = proof.commit_phase_openings[0]
    cidx = proof.commit_phase_indices[0]
    sites = {"trace cap": 5, "quotient cap": 1 + 32 * len(proof.trace_commit) + 5,
             "trace_local": raw.index(b(proof.trace_local)[:16]) + 1,
             "quotient chunk": raw.index(b(proof.quotient_chunks[0])[:16]) + 2,
             "commit-phase cap": raw.index(b(proof.commit_phase_commits[0])[:32]) + 3,
             "opened row": raw.index(b(np.asarray(rows[0]).reshape(len(idx), -1)[0])[:16]) + 1,
             "input path": raw.index(b(prune_paths(idx, paths)[:1])) + 7,
             "commit-phase sibling": raw.index(b(np.asarray(sib).reshape(len(cidx), -1)[0])[:16]) + 1,
             "commit-phase path": raw.index(b(prune_paths(cidx, cpaths)[:1])) + 9,
             "final poly": raw.index(b(proof.final_poly)[:16]) + 1,
             "query pow witness": len(raw) - 4, "degree_bits": len(raw) - 1}
    return sites


def _check(config, vcfg, air, raw, proof, **kw):
    verify(config, air, raw, **kw)
    verify(vcfg, air, raw, **kw)                                   # no product hashing: hashlib MMCS, restated transcript
    for name, pos in _sections(raw, proof).items():
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(config, air, bytes(bad), **kw)
            pytest.fail(f"a flipped byte in the {name} was accepted")


NEW_BENCHMARK = (1, 0, 1, 100, 0, 16)                                # FriParameters::new_benchmark


@pytest.mark.parametrize("node", sorted(KINDS))
def test_reference_example_statement(gpu, node):
    """prove_baby_bear_sha256(_compress).rs: KeccakAir over BabyBear, 1,365 hashes (a 2^15-row trace), new_benchmark, cap 3."""
    from plonky3_b200 import keccak_air
    f = BabyBear
    config = _config(gpu, f, node, NEW_BENCHMARK, 3)
    air = keccak_air.KeccakAir(f, gpu)
    trace = air.generate_trace_rows(torch.from_numpy(keccak_air.random_inputs(1365).view(np.int64)).cuda())
    assert tuple(trace.shape) == (1 << 15, 2633)
    proof = prove(config, air, trace)
    assert proof.digest_codec == DIGEST_U8X32 and proof.degree_bits == 15
    raw = proof.to_postcard()
    _check(config, S.verifier_config(f, node, NEW_BENCHMARK), keccak_air.KeccakAir(f), raw, proof)
    assert prove(config, air, trace).to_postcard() == raw          # deterministic, smallest witnesses


def test_koala_bear_keccak_air(gpu):
    from plonky3_b200 import keccak_air
    f, node, fri = KoalaBear, "compress", (1, 0, 3, 40, 0, 8)
    config = _config(gpu, f, node, fri, 3)
    air = keccak_air.KeccakAir(f, gpu)
    trace = air.generate_trace_rows(torch.from_numpy(keccak_air.random_inputs(170).view(np.int64)).cuda())
    proof = prove(config, air, trace)
    raw = proof.to_postcard()
    _check(config, S.verifier_config(f, node, fri), keccak_air.KeccakAir(f), raw, proof)


@pytest.mark.parametrize("node", sorted(KINDS))
def test_fibonacci_dsl_air_with_public_values(gpu, node, monkeypatch):
    import air_examples as E
    from plonky3_b200.air import SymbolicAir
    from test_air_preprocessed_cpu import LayoutMockGpu
    f, n, fri = KoalaBear, 1 << 6, (2, 1, 2, 20, 0, 6)
    config = _config(gpu, f, node, fri, 1)
    trace = E.fib_trace(f, n)
    pis = [0, 1, f.from_monty(int(trace[-1, 1]))]
    air = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    proof = prove(config, air, dev(trace), pis)
    raw = proof.to_postcard()
    _check(config, S.verifier_config(f, node, fri), air, raw, proof, public_values=pis)
    with pytest.raises(VerificationError):
        verify(config, air, raw, pis[:2] + [pis[2] + 1])
    mock = S.with_sha256(LayoutMockGpu)()                          # the stand-in device (hashlib MMCS) writes the same bytes
    mair = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=mock)
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        assert prove(S.mock_config(f, mock, node, fri, 1), mair, torch.from_numpy(trace.view(np.int32)), pis).to_postcard() == raw


def test_preprocessed_and_periodic_air(gpu):
    from test_air_preprocessed_cpu import _air_and_trace
    log_n, fri, node = 5, (1, 1, 1, 12, 0, 5), "hasher"
    config = _config(gpu, BabyBear, node, fri, 2)
    air, trace = _air_and_trace("mixed", 1 << log_n, gpu)
    data, vk = setup_preprocessed(config, air, log_n)
    proof = prove(config, air, dev(trace), preprocessed=data)
    assert proof.preprocessed_local is not None
    raw = proof.to_postcard()
    _check(config, S.verifier_config(BabyBear, node, fri), air, raw, proof, preprocessed_vk=vk)


# ---------------------------------------------------------------- the row-sharded prove
def _sharded_rank(gpu, rank, world, node, field_name):
    from plonky3_b200 import sha256_air
    from plonky3_b200.distributed import PeerGroup, column_starts, prove_sharded
    f = {"bb": BabyBear, "kb": KoalaBear}[field_name]
    log_n = 12                                                     # the sharded LDE's tiled path needs 2^12 rows
    m = MerkleTreeMmcs.sha256(f, cap_height=3, gpu=gpu, node=node)
    config = Sha256StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)))
    air = sha256_air.Sha256Air(f, gpu)
    inputs = torch.from_numpy(np.ascontiguousarray(sha256_air.random_inputs(1 << log_n)).view(np.int32)).to(f"cuda:{gpu.device}")
    full = air.generate_trace_rows(inputs)
    starts = column_starts(air.width(), world, align=8)
    block = air.generate_trace_cols(inputs, starts[rank], starts[rank + 1])
    grp = PeerGroup(gpu, (2 << log_n) // world, air.width(), timeout_s=60.0)
    try:
        expected = prove(config, air, full).to_postcard()
        raw = prove_sharded(config, air, grp, block, starts).to_postcard()
        bad = [] if raw == expected else ["prove_sharded bytes differ from prove"]
        if rank == 0:
            verify(config, air, raw)
    finally:
        grp.close()
    return bad


def _rank_main(rank, world, port, node, field_name, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        import torch.distributed as dist
        device = rank if torch.cuda.device_count() >= world else 0
        torch.cuda.set_device(device)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        bad = _sharded_rank(Gpu(device), rank, world, node, field_name)
        q.put((rank, not bad, "; ".join(bad)))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:                                       # noqa: BLE001 — surfaced by the parent
        import traceback
        q.put((rank, False, repr(e) + "\n" + traceback.format_exc()))


@pytest.mark.parametrize("node,field_name", [("hasher", "bb"), ("compress", "kb")])
def test_prove_sharded_single_rank_equals_prove(node, field_name):
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    assert not _sharded_rank(Gpu(0), 0, 1, node, field_name)


def test_prove_sharded_two_ranks_equal_prove():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29850 + (os.getpid() % 100)
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, "compress", "bb", q)) for r in range(world)]
    for p in procs: p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs: p.join(timeout=60)
    assert all(ok for _, ok, _ in res), "; ".join(f"rank {r}: {m}" for r, ok, m in sorted(res) if not ok)
