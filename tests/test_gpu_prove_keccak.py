"""The Keccak configuration on the GPU (uni_stark.KeccakStarkConfig: Keccak MMCS, SerializingChallenger32 over Keccak-256 resident on
the device): the device transcript equals the restatement (tests/keccak_transcript.py) on random observe/sample scripts over both
fields, host and device inputs and clones; the grinding kernel returns the sequential smallest witness; the config-5 AIR, the DSL
Fibonacci AIR with public values and an AIR with preprocessed and periodic columns prove with the bytes of the same driver on the
oracle-backed stand-in device, and both verifiers accept them and reject corruptions."""
import numpy as np
import pytest
import torch

import keccak_transcript as K
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200.challenger import SerializingChallenger32
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.proof_io import DIGEST_U64X4
from plonky3_b200.uni_stark import KeccakStarkConfig, VectorizedPoseidon2Air, prove, setup_preprocessed, verify
from plonky3_b200.verifier import VerificationError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


# ---------------------------------------------------------------- the transcript
@pytest.mark.parametrize("field", [BabyBear, KoalaBear])
def test_device_transcript_matches_restatement(gpu, field):
    rng = np.random.default_rng(17 + field.id)
    ch, rs = SerializingChallenger32.from_hasher([], field, gpu), K.SerializingChallenger32.from_hasher(field)
    pairs = [(ch, rs)]
    for step in range(120):
        d, r = pairs[rng.integers(0, len(pairs))]
        op = rng.integers(0, 7)
        if op == 0:                                                # host field elements, across block boundaries
            v = rng.integers(0, field.P, int(rng.integers(0, 80)), dtype=np.uint32)
            d.observe_slice(v); r.observe_slice(v)
        elif op == 1:                                              # device-resident field elements
            v = rng.integers(0, field.P, int(rng.integers(1, 300)), dtype=np.uint32)
            d.observe_slice(dev(v)); r.observe_slice(v)
        elif op == 2:                                              # a cap of [u64; 4] digests: any 32-bit words
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


def test_device_transcript_rejects_bad_input_before_launch(gpu):
    ch = SerializingChallenger32.from_hasher([], KoalaBear, gpu)
    n0 = gpu.launches
    for bits in (31, 32, 40):
        with pytest.raises(_lib.P3GpuError) as ex:
            ch.sample_bits(bits)
        assert ex.value.code == _lib.EINVAL
        with pytest.raises(_lib.P3GpuError) as ex:
            ch.grind(bits)
        assert ex.value.code == _lib.EINVAL
    with pytest.raises(_lib.P3GpuError) as ex:
        ch.observe(KoalaBear.P)                                    # not a canonical Montgomery word
    assert ex.value.code == _lib.EINVAL
    assert gpu.launches == n0
    assert ch.grind(0) == 0 and gpu.launches == n0                 # 0 bits: no witness search, the state untouched
    rs = K.SerializingChallenger32.from_hasher(KoalaBear)
    assert list(ch.sample_many(3)) == list(rs.sample_many(3))


@pytest.mark.parametrize("field", [BabyBear, KoalaBear])
def test_grind_returns_the_sequential_smallest_witness(gpu, field):
    """Pending tails of 0, 8, 33 (the candidate completes the block, the padding needs a second one) and 20 words."""
    rng = np.random.default_rng(5)
    for bits in range(1, 17):
        ch, rs = SerializingChallenger32.from_hasher([], field, gpu), K.SerializingChallenger32.from_hasher(field)
        prefix = [0, 34, 33, 34 * 3 + 20][bits % 4]
        v = rng.integers(0, field.P, prefix, dtype=np.uint32)
        ch.observe_slice(v); rs.observe_slice(v)
        if bits % 5 == 0:                                          # after a flush: the digest is the pending input
            assert ch.sample() == rs.sample()
        w = ch.grind(bits)
        assert w == rs.grind(bits), bits
        assert list(ch.sample_many(2)) == list(rs.sample_many(2))
    ch, rs = SerializingChallenger32.from_hasher([], field, gpu), K.SerializingChallenger32.from_hasher(field)
    v = rng.integers(0, field.P, 57, dtype=np.uint32)
    ch.observe_slice(v); rs.observe_slice(v)
    w = ch.grind(20)
    assert rs.clone().check_witness(20, w)
    assert rs.check_witness(20, w) and list(ch.sample_many(4)) == list(rs.sample_many(4))


# ---------------------------------------------------------------- proofs
def _configs(gpu, mock, field, fri, cap_height):
    """The same configuration on the GPU (KeccakStarkConfig) and on the stand-in device (restated transcript), and the product
    verifier's configuration with oracle stand-ins."""
    from types import SimpleNamespace
    mk = lambda g: MerkleTreeMmcs.keccak(field, cap_height=cap_height, gpu=g)
    m_gpu = mk(gpu)
    config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m_gpu, FriParameters(*fri, m_gpu)))
    if mock is None:
        return config, None, None
    m_mock = mk(mock)
    mconfig = SimpleNamespace(pcs=TwoAdicFriPcs(Radix2DitParallel(field, mock), m_mock, FriParameters(*fri, m_mock)), digest_codec="u64x4",
                              initialise_challenger=lambda: K.SerializingChallenger32.from_hasher(field))
    vcfg = K.verifier_config(field, fri[3], fri[5], log_blowup=fri[0], log_final_poly_len=fri[1], max_log_arity=fri[2])
    return config, mconfig, vcfg


def _check_rejections(config, air, raw, proof, **kw):
    """A flipped byte in the trace cap, an opened value, a pruned sibling hash, the query proof-of-work witness."""
    from plonky3_b200.merkle_tree import prune_paths
    from plonky3_b200.proof_io import _vec_of_digests
    cap = len(_vec_of_digests(proof.trace_commit, DIGEST_U64X4))
    qcap = len(_vec_of_digests(proof.quotient_commit, DIGEST_U64X4))
    (rows, paths), idx = proof.input_openings[0], proof.input_opening_indices[0]
    sib = _vec_of_digests(prune_paths(idx, paths)[:1], DIGEST_U64X4)[1:]
    sites = [3, cap + qcap + 4, raw.index(sib) + 1, len(raw) - 6]
    for pos in sites:
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(config, air, bytes(bad), **kw)


P2_FRI = (1, 0, 3, 100, 0, 16)                                      # new_benchmark_high_arity


@pytest.mark.parametrize("log_perms", [10, 12, 14])
def test_config5_air_proves_and_verifies(gpu, log_perms, monkeypatch):
    import mock_device as M
    f, log_rows = KoalaBear, log_perms - 3
    mock = M.MockGpu()
    config, mconfig, vcfg = _configs(gpu, mock, f, P2_FRI, 3)
    oair = K.p2_air_setup(f)
    air = VectorizedPoseidon2Air(f, K.p2_round_constants(oair), gpu)
    inputs = K.p2_inputs(f, log_rows)
    proof = prove(config, air, air.generate_trace_rows(dev(inputs)))
    assert proof.degree_bits == log_rows and proof.digest_codec == DIGEST_U64X4
    raw = proof.to_postcard()
    verify(config, air, raw)
    verify(vcfg, air, raw)
    _check_rejections(config, air, raw, proof)
    if log_perms == 10:                                            # the stand-in device writes the same bytes
        mair = VectorizedPoseidon2Air(f, K.p2_round_constants(oair), mock)
        with monkeypatch.context() as mp:
            mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
            mraw = prove(mconfig, mair, mair.generate_trace_rows(torch.from_numpy(inputs.view(np.int32)))).to_postcard()
        assert mraw == raw


def test_fibonacci_dsl_air_with_public_values(gpu, monkeypatch):
    import air_examples as E
    from plonky3_b200.air import SymbolicAir
    from test_air_preprocessed_cpu import LayoutMockGpu
    f, n = BabyBear, 1 << 6
    mock = LayoutMockGpu()
    fri = (2, 1, 2, 20, 0, 6)
    config, mconfig, vcfg = _configs(gpu, mock, f, fri, 1)
    trace = E.fib_trace(f, n)
    pis = [0, 1, f.from_monty(int(trace[-1, 1]))]
    air = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=gpu)
    proof = prove(config, air, dev(trace), pis)
    raw = proof.to_postcard()
    verify(config, air, raw, pis)
    verify(vcfg, air, raw, pis)
    with pytest.raises(VerificationError):
        verify(config, air, raw, pis[:2] + [pis[2] + 1])
    _check_rejections(config, air, raw, proof, public_values=pis)
    mair = SymbolicAir(f, 2, E.fib_eval, num_public_values=3, gpu=mock)
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        assert prove(mconfig, mair, torch.from_numpy(trace.view(np.int32)), pis).to_postcard() == raw


def test_preprocessed_and_periodic_air(gpu, monkeypatch):
    from test_air_preprocessed_cpu import LayoutMockGpu, _air_and_trace
    log_n = 5
    mock = LayoutMockGpu()
    fri = (1, 1, 1, 12, 0, 5)
    config, mconfig, vcfg = _configs(gpu, mock, BabyBear, fri, 2)
    air, trace = _air_and_trace("mixed", 1 << log_n, gpu)
    data, vk = setup_preprocessed(config, air, log_n)
    proof = prove(config, air, dev(trace), preprocessed=data)
    assert proof.preprocessed_local is not None
    raw = proof.to_postcard()
    verify(config, air, raw, preprocessed_vk=vk)
    verify(vcfg, air, raw, preprocessed_vk=vk)
    _check_rejections(config, air, raw, proof, preprocessed_vk=vk)
    mair, _ = _air_and_trace("mixed", 1 << log_n, mock)
    mdata, _ = setup_preprocessed(mconfig, mair, log_n)
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        assert prove(mconfig, mair, torch.from_numpy(trace.view(np.int32)), preprocessed=mdata).to_postcard() == raw


def test_config5_shape_at_2_20_permutations(gpu):
    f, log_rows = KoalaBear, 17
    config, _, _ = _configs(gpu, None, f, P2_FRI, 3)
    air = VectorizedPoseidon2Air(f, K.p2_round_constants(K.p2_air_setup(f)), gpu)
    g = torch.Generator(device="cuda"); g.manual_seed(20)
    inputs = torch.randint(0, f.P, (8 << log_rows, 16), device="cuda", dtype=torch.int32, generator=g)
    proof = prove(config, air, air.generate_trace_rows(inputs))
    verify(config, air, proof.to_postcard())
