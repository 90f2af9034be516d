"""The SHA-256 AIR's kernels on the GPU (csrc/sha256_air.cu): the trace equals the restated generation bit for bit on a poisoned
buffer; the quotient equals the constraint-DAG oracle on valid-trace and random LDEs, and is a polynomial of degree < 2N - 2 on a
valid trace only; bad arguments are refused before any launch; proofs under both configurations have the stand-in device's bytes
and pass the verifier; the reference bench's configuration proves and verifies at 2^12 compressions; the 2^18-row shape proves and
verifies."""
import numpy as np
import pytest
import torch

import air_oracle as A
import sha256_air_oracle as SO
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200 import sha256_air as SA
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_keccak_air_cpu import corruption_sites, poseidon2_setup
from test_sha256_air_cpu import FIELDS, NUM_QUERIES, POW_BITS, PROOF_CASES, _edge_inputs, _inputs, mock_prove

pytestmark = pytest.mark.gpu
POISON = -1                                                            # 0xffffffff: above p in both fields


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def _dev_inputs(inputs):
    return torch.from_numpy(np.ascontiguousarray(inputs, dtype=np.uint32).view(np.int32)).cuda()


def _gen_poisoned(gpu, field, inputs):
    n = inputs.shape[0]
    x = _dev_inputs(inputs)
    out = torch.full((n + 1, SA.WIDTH), POISON, dtype=torch.int32, device="cuda")      # one guard row
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_sha256_air_generate_trace_dev(gpu.h, field.id, x.data_ptr(), n, out.data_ptr()))
    torch.cuda.synchronize()
    assert bool((out[-1] == POISON).all()), "write past the trace"
    return out[:-1]


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("n", [1, 2, 32, 1024, 16384])
def test_trace_matches_the_oracle(gpu, field, n):
    inputs = _edge_inputs(n, 50 + n)
    got = _gen_poisoned(gpu, field, inputs)
    assert got.shape == (n, SA.WIDTH)
    step = 2048
    for h0 in range(0, n, step):                                         # compare in chunks of rows
        h1 = min(n, h0 + step)
        exp = SO.generate_rows(field.id, inputs[h0:h1])
        assert np.array_equal(got[h0:h1].cpu().numpy().view(np.uint32), exp), (h0, h1)
    if n == 32:                                                          # the generate_trace_rows wrapper writes the same
        w = SA.Sha256Air(field, gpu).generate_trace_rows(_dev_inputs(inputs))
        assert torch.equal(w, got)


def _lde(gpu, field, trace_np, log_blowup):
    t = torch.from_numpy(np.ascontiguousarray(trace_np, dtype=np.uint32).view(np.int32)).cuda()
    return gpu.coset_lde_batch(field.id, t, log_blowup, field.generator, bitrev_rows=True)


@pytest.mark.parametrize("field", FIELDS)
def test_quotient_matches_the_dag_oracle(gpu, field):
    nodes, cons = SO.air_dag(field)
    rng = np.random.default_rng(7 + field.id)
    for log_n in range(2, 11):
        valid = SO.generate(field.id, _edge_inputs(1 << log_n, log_n))
        rand = rng.integers(0, field.P, (1 << log_n, SA.WIDTH), dtype=np.uint32)
        for log_blowup in (1, 2):
            for kind, tr in (("valid", valid), ("random", rand)):
                lde = _lde(gpu, field, tr, log_blowup)
                alpha = rng.integers(0, field.P, 4, dtype=np.uint32)
                q = gpu.sha256_air_quotient(field.id, lde, log_n, alpha).cpu().numpy().view(np.uint32)
                exp = A.air_quotient(field.id, nodes, cons, lde.cpu().numpy().view(np.uint32), log_n + 1, log_n, [], alpha)
                assert np.array_equal(q, exp), (log_n, log_blowup, kind)
                if log_blowup == 1:
                    # coefficients over the coset: degree <= 3 (N - 1) - N = 2N - 3 exactly when the trace satisfies the AIR
                    coeffs = O.coset_idft_batch(field.id, q, field.generator)
                    assert (not np.any(coeffs[(2 << log_n) - 2:])) == (kind == "valid"), (log_n, kind)


def test_bad_arguments_are_refused_before_launch(gpu):
    f = KoalaBear
    lde = _lde(gpu, f, SO.generate(f.id, _inputs(32, 1)), 1)              # 2^6 rows over a 2^5-row trace
    q = torch.empty((64, 4), dtype=torch.int32, device="cuda")
    al = np.array([1, 2, 3, 4], dtype=np.uint32)
    L, h = gpu.L, gpu.h
    torch.cuda.synchronize()
    n0 = gpu.launches
    cases = [
        ((h, f.id, None, 6, 5, al.ctypes.data, q.data_ptr()), _lib.EINVAL),
        ((h, f.id, lde.data_ptr(), 6, 5, None, q.data_ptr()), _lib.EINVAL),
        ((h, f.id, lde.data_ptr(), 6, 5, al.ctypes.data, None), _lib.EINVAL),
        ((h, f.id, lde.data_ptr() + 2, 6, 5, al.ctypes.data, q.data_ptr()), _lib.EINVAL),
        ((h, f.id, lde.data_ptr(), 6, 5, al.ctypes.data, q.data_ptr() + 1), _lib.EINVAL),
        ((h, f.id, lde.data_ptr(), 6, 6, al.ctypes.data, q.data_ptr()), _lib.EINVAL),        # log_trace_height + 1 > log_lde_height
        ((h, f.id, lde.data_ptr(), 30, 5, al.ctypes.data, q.data_ptr()), _lib.EINVAL),       # above the two-adicity
        ((h, f.id, lde.data_ptr(), 6, 5, np.array([f.P, 0, 0, 0], np.uint32).ctypes.data, q.data_ptr()), _lib.EINVAL),   # alpha >= p
        ((h, 7, lde.data_ptr(), 6, 5, al.ctypes.data, q.data_ptr()), _lib.EUNSUPPORTED),
    ]
    for args, code in cases:
        assert L.p3gpu_sha256_air_quotient_dev(*args) == code, args
    x = torch.zeros((4, 24), dtype=torch.int32, device="cuda")
    t = torch.empty((4, SA.WIDTH), dtype=torch.int32, device="cuda")
    gen = L.p3gpu_sha256_air_generate_trace_dev
    assert gen(h, f.id, None, 4, t.data_ptr()) == _lib.EINVAL
    assert gen(h, f.id, x.data_ptr(), 4, None) == _lib.EINVAL
    assert gen(h, f.id, x.data_ptr() + 2, 4, t.data_ptr()) == _lib.EINVAL
    assert gen(h, f.id, x.data_ptr(), 4, t.data_ptr() + 2) == _lib.EINVAL
    assert gen(h, f.id, x.data_ptr(), 0, t.data_ptr()) == _lib.EINVAL                     # no hashes
    assert gen(h, f.id, x.data_ptr(), 3, t.data_ptr()) == _lib.EINVAL                     # not a power of two
    assert gen(h, 7, x.data_ptr(), 4, t.data_ptr()) == _lib.EUNSUPPORTED
    assert gpu.launches == n0


def _gpu_config(gpu, field, config_name):
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig
    if config_name == "keccak":
        m = MerkleTreeMmcs.keccak(field, cap_height=3, gpu=gpu)
        return KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m, FriParameters(1, 0, 3, NUM_QUERIES, 0, POW_BITS, m)))
    return poseidon2_setup(field, gpu, NUM_QUERIES, POW_BITS, device_challenger=True)[0]


@pytest.mark.parametrize("field,config_name,n_hashes", PROOF_CASES)
def test_gpu_proofs_have_the_stand_in_bytes(gpu, monkeypatch, field, config_name, n_hashes):
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4
    from plonky3_b200.uni_stark import prove, verify
    from plonky3_b200.verifier import VerificationError
    config = _gpu_config(gpu, field, config_name)
    air = SA.Sha256Air(field, gpu)
    proof = prove(config, air, air.generate_trace_rows(_dev_inputs(_edge_inputs(n_hashes, 7))))
    raw = proof.to_postcard()
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        _, mraw, vcfg = mock_prove(field, config_name, n_hashes)
    assert raw == mraw
    verify(vcfg, SA.Sha256Air(field), raw)
    verify(config, air, raw)                                             # the product verifier with the device transcript
    for pos in corruption_sites(raw, proof, DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, SA.Sha256Air(field), bytes(bad))


def _keccak_config(gpu, field, params):
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.uni_stark import KeccakStarkConfig
    m = MerkleTreeMmcs.keccak(field, cap_height=3, gpu=gpu)
    return KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(field, gpu), m, getattr(FriParameters, params)(m)))


def test_the_reference_bench_configuration_at_2_12_compressions(gpu):
    """sha256-air/benches/sha256-air.rs: BabyBear, the Keccak MMCS with cap height 3, the Keccak-256 transcript and
    FriParameters::new_benchmark, at 2^12 compressions of Sha256Air::generate_trace_rows' draw."""
    from plonky3_b200.uni_stark import prove, verify
    f, n = BabyBear, 1 << 12
    config = _keccak_config(gpu, f, "new_benchmark")
    air = SA.Sha256Air(f, gpu)
    proof = prove(config, air, air.generate_random_trace_rows(n))
    assert proof.degree_bits == 12 and len(proof.quotient_chunks) == 2
    verify(config, SA.Sha256Air(f), proof.to_postcard())


def test_full_shape_at_2_18_rows(gpu):
    """2^18 compressions (a 2^18 x 7728 trace, 8.1 GB; its LDE 16.2 GB), KoalaBear, the Keccak configuration with
    new_benchmark_high_arity and cap height 3."""
    from plonky3_b200.uni_stark import prove, verify
    f, n = KoalaBear, 1 << 18
    config = _keccak_config(gpu, f, "new_benchmark_high_arity")
    air = SA.Sha256Air(f, gpu)
    trace = air.generate_random_trace_rows(n)
    assert tuple(trace.shape) == (n, SA.WIDTH)
    inputs = SA.random_inputs(n)
    for r in (0, n - 1):
        exp = SO.generate_rows(f.id, inputs[r:r + 1])
        assert np.array_equal(trace[r:r + 1].cpu().numpy().view(np.uint32), exp), r
    proof = prove(config, air, trace)
    del trace
    torch.cuda.empty_cache()
    verify(config, SA.Sha256Air(f), proof.to_postcard())
