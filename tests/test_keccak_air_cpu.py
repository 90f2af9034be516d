"""The Keccak-f AIR (plonky3_b200.keccak_air) without a GPU: its column layout, the restated trace generation
(tests/keccak_air_oracle.py) against the pinned Keccak-f, the constraint DAG (count, degree, vanishing on valid traces over both
fields, and the corruptions of keccak-air/src/air.rs's unit tests), and proofs on the oracle-backed stand-in device under both
configurations, accepted by the product verifier and the restated one and rejecting tampered bytes."""
import copy

import numpy as np
import pytest
import torch

import air_oracle as A
import keccak_air_oracle as KO
import mock_device as M
from oracle import p3_oracle as O
from plonky3_b200 import keccak_air as KA
from plonky3_b200.field import BabyBear, KoalaBear

FIELDS = [BabyBear, KoalaBear]


def _inputs(n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 1 << 64, (n, 25), dtype=np.uint64)


class KeccakMockGpu(M.MockGpu):
    """The stand-in device with the Keccak AIR's two calls: the trace from the restated generation, the quotient from the
    constraint-DAG oracle (tests/air_oracle.py) on the AIR's DAG."""

    def keccak_air_generate_trace(self, field, inputs):
        self._note("keccak_air_generate_trace")
        return M._t(KO.generate(field, inputs.contiguous().numpy().view(np.uint64)))

    def keccak_air_quotient(self, field, lde, log_trace_height, alpha):
        self._note("keccak_air_quotient")
        nodes, cons = KO.air_dag(BabyBear if field == BabyBear.id else KoalaBear)
        return M._t(A.air_quotient(field, nodes, cons, M._n(lde), log_trace_height + 1, log_trace_height, [], M._n(alpha)))


# ---------------------------------------------------------------- layout, trace, constraints
def test_width_and_column_offsets():
    assert KA.WIDTH == 2633
    air = KA.KeccakAir(KoalaBear)
    assert air.width() == 2633 and air.num_public_values() == 0 and air.main_next_row_columns() == list(range(2633))
    assert (KA.STEP_FLAGS, KA.EXPORT, KA.PREIMAGE, KA.A, KA.C, KA.C_PRIME, KA.A_PRIME) == (0, 24, 25, 125, 225, 545, 865)
    assert (KA.A_PRIME_PRIME, KA.A_PRIME_PRIME_0_0_BITS, KA.A_PRIME_PRIME_PRIME_0_0_LIMBS) == (2465, 2565, 2629)
    assert KA.preimage(4, 4, 3) == 124 and KA.a(4, 4, 3) == 224 and KA.c(4, 63) == 544 and KA.c_prime(4, 63) == 864
    assert KA.a_prime(4, 4, 63) == 2464 and KA.a_prime_prime(4, 4, 3) == 2564
    # the constraints read only step_flags, preimage and a of the next row
    assert max(int(n[1]) for n in air.nodes if n[0] == KO.MAIN_NEXT) == KA.NEXT_ROW_READ - 1


@pytest.mark.parametrize("field", FIELDS)
def test_oracle_trace_matches_keccak_f_and_pads_with_the_zero_block(field):
    edge = np.array([[0] * 25, [(1 << 64) - 1] * 25], dtype=np.uint64)
    for n, inputs in ((0, np.zeros((0, 25), np.uint64)), (1, edge[1:]), (3, np.vstack([edge, _inputs(1, 3)])), (6, _inputs(6, 4))):
        tr = KO.generate(field.id, inputs)
        H = KO.height(n)
        assert tr.shape == (H, 2633) and H == (1 if n == 0 else 1 << (24 * n - 1).bit_length())
        for i in range(n):
            assert np.array_equal(KO.output_state(field.id, tr, i), O.keccak_f(inputs[i])), (n, i)
        zero = KO.perm_rows(field.id, np.zeros((1, 25), np.uint64))[0]
        for r in range(24 * n, H):
            assert np.array_equal(tr[r], zero[(r - 24 * n) % 24]), r
        assert np.all(tr < field.P)


def test_random_inputs_are_fixed_seed_and_deterministic():
    a, b = KA.random_inputs(3), KA.random_inputs(3)
    assert a.shape == (3, 25) and a.dtype == np.uint64 and np.array_equal(a, b)
    assert np.array_equal(KA.random_inputs(5)[:3], a)
    import fixture_replay as FR
    rng = FR.SmallRng(1)                                              # the pinned u32 draw is the high half of the u64 draw
    assert [int(v) >> 32 for v in a.ravel()[:6]] == [rng.u32() for _ in range(6)]


@pytest.mark.parametrize("field", FIELDS)
def test_constraint_count_and_degree(field):
    air = KA.KeccakAir(field)
    degs = air.constraint_degrees()
    assert len(degs) == 3182 and max(degs) == 3 and air.max_constraint_degree() == 3


@pytest.mark.parametrize("field", FIELDS)
def test_constraints_vanish_on_every_row_of_valid_traces(field):
    nodes, cons = KO.air_dag(field)
    for n, seed in ((1, 10), (2, 11), (5, 12)):                      # 2 and 5 cross the row-23 -> row-24 boundary
        tr = KO.generate(field.id, _inputs(n, seed))
        assert not np.any(KO.constraint_values(field.id, nodes, cons, tr))
    tr = KO.generate(field.id, np.array([[(1 << 64) - 1] * 25, [0] * 25], dtype=np.uint64))
    assert not np.any(KO.constraint_values(field.id, nodes, cons, tr))


def _violated(field, tr):
    nodes, cons = KO.air_dag(field)
    return bool(np.any(KO.constraint_values(field.id, nodes, cons, tr)))


@pytest.mark.parametrize("field", FIELDS)
def test_reference_corruptions_are_detected(field):
    """keccak-air/src/air.rs tests: every mutation of the zero-input trace breaks some constraint."""
    one = field.to_monty(1)
    base = KO.generate(field.id, np.zeros((1, 25), np.uint64))

    def flip(v): return 0 if int(v) else one

    def add1(v): return field.to_monty((field.from_monty(int(v)) + 1) % field.P)
    cases = [
        [(0, KA.STEP_FLAGS, lambda v: 0), (0, KA.STEP_FLAGS + 1, lambda v: one)],
        [(1, KA.preimage(0, 0, 0), lambda v: field.to_monty(0xBEEF))],
        [(0, KA.c(0, 0), lambda v: field.to_monty(2))],
        [(0, KA.a_prime(0, 0, 0), flip)],
        [(0, KA.a_prime_prime(0, 0, 0), add1)],
        [(0, KA.A_PRIME_PRIME_0_0_BITS, flip)],
        [(0, KA.A_PRIME_PRIME_PRIME_0_0_LIMBS, add1)],
        [(1, KA.a(0, 0, 0), add1)],
    ]
    for case in cases:
        tr = base.copy()
        for row, col, fn in case:
            tr[row, col] = fn(tr[row, col])
        assert _violated(field, tr), case


@pytest.mark.parametrize("field", FIELDS)
def test_single_bit_flips_in_c_and_a_prime_are_detected(field):
    rng = np.random.default_rng(99 + field.id)
    one = field.to_monty(1)
    for t in range(12):
        tr = KO.generate(field.id, _inputs(1, 100 + t))
        col = (KA.c(int(rng.integers(5)), int(rng.integers(64))) if t % 2 == 0
               else KA.a_prime(int(rng.integers(5)), int(rng.integers(5)), int(rng.integers(64))))
        tr[0, col] = 0 if int(tr[0, col]) else one
        assert _violated(field, tr), col


# ---------------------------------------------------------------- proofs on the stand-in device
def poseidon2_setup(field, gpu, num_queries, pow_bits, device_challenger=False):
    """The Poseidon2 configuration's shape (DuplexChallenger, Poseidon2 MMCS, log_blowup 1, arity 8) on `gpu` (a real device or
    the stand-in), with the transcript on the host oracle (device_challenger: uni_stark.StarkConfig, the transcript on the
    device, the same sponge); and the restated verifier's dict configuration.  BabyBear: the
    reference Fibonacci fixture's Poseidon2-16 (rate 8); KoalaBear: the example binary's Poseidon2-16 / -24 (rate 16)."""
    from types import SimpleNamespace
    import p2_prove_replay as R
    from plonky3_b200.dft import Radix2DitParallel
    from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
    from plonky3_b200.merkle_tree import MerkleTreeMmcs
    from plonky3_b200.poseidon2 import Poseidon2
    if field is BabyBear:
        import fixture_replay as FR
        from test_air_program_cpu import BabyBearChallenger
        rc_i, rc_t, rc_p = FR.fixture_constants()
        pm = Poseidon2.new(BabyBear, 16, rc_i, rc_t, rc_p, monty=True)
        mmcs = MerkleTreeMmcs.poseidon2(pm, None, 0, gpu)
        operm = O.make_perm(BabyBear.id, 16, rc_i, rc_t, rc_p, monty=True)
        chal, perm, rate = (lambda: BabyBearChallenger(operm)), pm, 8
        cfg = dict(hasher=O.poseidon2_hasher(operm, operm), challenger_perm=operm, challenger_width=16, challenger_rate=8)
    else:
        rng = O.SmallRng(1)
        O.air_from_rng(field.id, rng)
        o16, o24 = O.perm_from_rng(field.id, 16, rng), O.perm_from_rng(field.id, 24, rng)
        mk = lambda pm: Poseidon2.new(field, pm.width, np.array(pm.rc_init)[: 4 * pm.width].reshape(4, pm.width),
                                      np.array(pm.rc_term)[: 4 * pm.width].reshape(4, pm.width), np.array(pm.rc_int)[: pm.rounds_p], monty=True)
        p24 = mk(o24)
        mmcs = MerkleTreeMmcs.poseidon2(mk(o16), p24, cap_height=3, gpu=gpu)
        chal, perm, rate = (lambda: M.MockChallenger(o24)), p24, 16
        cfg = R.verifier_config(o16, o24)
    cfg.update(log_blowup=1, log_final_poly_len=0, max_log_arity=3, num_queries=num_queries, commit_pow_bits=0, query_pow_bits=pow_bits)
    pcs = TwoAdicFriPcs(Radix2DitParallel(field, gpu), mmcs, FriParameters(1, 0, 3, num_queries, 0, pow_bits, mmcs))
    if device_challenger:
        from plonky3_b200.uni_stark import StarkConfig
        return StarkConfig(pcs, perm, rate), cfg
    return SimpleNamespace(pcs=pcs, initialise_challenger=chal), cfg


def restated_air(field):
    """The restated verifier's AIR dict (tests/stark_verify.py) folding the Keccak AIR's DAG in its own arithmetic."""
    nodes, cons = KO.air_dag(field)

    def constraints(f, loc, nxt, pis, is_first, is_last, is_trans, alpha):
        sel = {KO.IS_FIRST_ROW: is_first, KO.IS_LAST_ROW: is_last, KO.IS_TRANSITION: is_trans}
        vals = []
        for op, a, b, imm in nodes.astype(np.int64):
            if op == KO.CONST:
                v = f.ebase(f.c(int(imm)))
            elif op == KO.MAIN_LOCAL:
                v = loc[a]
            elif op == KO.MAIN_NEXT:
                v = nxt[a]
            elif op in sel:
                v = sel[op]
            elif op == KO.ADD:
                v = f.eadd(vals[a], vals[b])
            elif op == KO.SUB:
                v = f.esub(vals[a], vals[b])
            elif op == KO.NEG:
                v = f.esub([0, 0, 0, 0], vals[a])
            else:
                v = f.emul(vals[a], vals[b])
            vals.append(v)
        acc = [0, 0, 0, 0]
        for k in cons:
            acc = f.eadd(f.emul(acc, alpha), vals[int(k)])
        return acc
    return {"width": KA.WIDTH, "main_next": True, "log_quotient_chunks": 1, "num_public_values": 0, "constraints": constraints}


def corruption_sites(raw, proof, codec):
    """Byte offsets in the trace cap, an opened value, the first pruned sibling hash of the trace batch, the query PoW witness."""
    from plonky3_b200.merkle_tree import prune_paths
    from plonky3_b200.proof_io import _vec_of_digests
    cap = len(_vec_of_digests(proof.trace_commit, codec))
    qcap = len(_vec_of_digests(proof.quotient_commit, codec))
    (rows, paths), idx = proof.input_openings[0], proof.input_opening_indices[0]
    sib = _vec_of_digests(prune_paths(idx, paths)[:1], codec)[1:]
    return [3, cap + qcap + 4, raw.index(sib) + 1, len(raw) - 6]


PROOF_CASES = [(f, c, n) for f in FIELDS for c in ("poseidon2", "keccak") for n in (5, 42)]   # 128 and 1024 rows
NUM_QUERIES, POW_BITS = 6, 3


def mock_prove(field, config_name, n_hashes):
    """(proof, raw bytes, KeccakAir on the stand-in, product verifier config, restated verifier args or None)."""
    import keccak_transcript as K
    import stark_verify as V
    from plonky3_b200.uni_stark import prove
    mock = KeccakMockGpu()
    if config_name == "keccak":
        config = K.keccak_mock_config(field, mock, NUM_QUERIES, POW_BITS)
        vcfg, restated = K.verifier_config(field, NUM_QUERIES, POW_BITS), None
    else:
        config, cfg = poseidon2_setup(field, mock, NUM_QUERIES, POW_BITS)
        vcfg, restated = V.product_config(field, cfg), (V.Fld(field.id), cfg, restated_air(field))
    air = KA.KeccakAir(field, mock)
    trace = air.generate_trace_rows(torch.from_numpy(_inputs(n_hashes, 7).view(np.int64)))
    proof = prove(config, air, trace)
    assert "keccak_air_quotient" in mock.calls
    return proof, proof.to_postcard(), air, vcfg, restated


@pytest.mark.parametrize("field,config_name,n_hashes", PROOF_CASES)
def test_proofs_on_the_stand_in_device(monkeypatch, field, config_name, n_hashes):
    import stark_verify as V
    from plonky3_b200.proof_io import DIGEST_F8, DIGEST_U64X4, proof_from_postcard
    from plonky3_b200.uni_stark import verify
    from plonky3_b200.verifier import VerificationError
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    proof, raw, air, vcfg, restated = mock_prove(field, config_name, n_hashes)
    assert proof.degree_bits == (24 * n_hashes - 1).bit_length() and len(proof.quotient_chunks) == 2
    assert proof.trace_next is not None and len(proof.trace_next) == 2633
    verifier_air = KA.KeccakAir(field)                                # verifier-only: no device
    verify(vcfg, verifier_air, raw)
    codec = DIGEST_U64X4 if config_name == "keccak" else DIGEST_F8
    if restated:
        V.verify(*restated[:2], restated[2], proof_from_postcard(raw))
    for pos in corruption_sites(raw, proof, codec):
        bad = bytearray(raw); bad[pos] ^= 1
        with pytest.raises(VerificationError):
            verify(vcfg, verifier_air, bytes(bad))
        if restated:
            with pytest.raises(V.VerifyError):
                V.verify(*restated[:2], restated[2], proof_from_postcard(bytes(bad)))
    # a proof of a trace that breaks a constraint is rejected at the out-of-domain check
    bad = copy.deepcopy(proof)
    bad.trace_local = np.array(bad.trace_local, dtype=np.uint32)
    bad.trace_local[KA.c(0, 0), 0] = (int(bad.trace_local[KA.c(0, 0), 0]) + 1) % field.P
    with pytest.raises(VerificationError):
        verify(vcfg, verifier_air, bad.to_postcard())
