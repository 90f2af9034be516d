"""The coset-blocked prove's host side, without a GPU: its refusals, its memory plan and the index identities it stands on.

CosetBlockedTrace (plonky3_b200/coset_blocks.py) refuses, before any device call and with a message naming the reason, the AIRs that
have no sharded quotient kernel (Keccak-f, BabyBear's Poseidon2), preprocessed columns, traces of fewer than 1024 rows, a configuration it does not know, a quotient
domain smaller than the LDE domain and a width the sharded quotient kernels' layout cannot take.  Its memory plan is twice the trace
plus a stated allowance.  Its blocks rest on three identities: memory rows [k N, (k+1) N) of the bit-reversed LDE are one coset (their
natural indices are congruent to bitrev(k) modulo the blowup), every point's next row lies in the same block, and the quotient slices
of the blocks, put back by `natural_order`, give the natural order."""
import types

import numpy as np
import pytest
import torch

import air_preprocessed_examples as PE
from plonky3_b200.air import SymbolicAir
from plonky3_b200.blake3_air import Blake3Air
from plonky3_b200.coset_blocks import (CosetBlockedTrace, coset_blocked_allowance_bytes, coset_blocked_error, coset_blocked_memory_bytes,
                                       prove_coset_blocked)
from plonky3_b200.distributed import _bitrev, natural_order, next_row_rank, quotient_slice_natural_indices
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.keccak_air import KeccakAir
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air
from plonky3_b200.sha256_air import Sha256Air
from plonky3_b200.uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig


class Untouchable:
    """A stand-in for the device and the trace: any use fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work before the refusal: .{name}")


def _pcs(log_blowup):
    """A PCS of which the refusals may read the blowup only."""
    return types.SimpleNamespace(fri=types.SimpleNamespace(log_blowup=log_blowup), dft=Untouchable(), mmcs=Untouchable())


def _poseidon2(field, rounds_p):
    rng = np.random.default_rng(5)
    return VectorizedPoseidon2Air(field, RoundConstants(rng.integers(0, field.P, (4, 16)), rng.integers(0, field.P, rounds_p),
                                                        rng.integers(0, field.P, (4, 16))), None)


def _fib(b):
    m = b.main()
    b.when_transition().assert_eq(m.local[1], m.next[0])
    b.assert_zero(m.local[0] * m.local[0] * m.local[1] - m.local[2])


CONFIGS = [StarkConfig(_pcs(1), None), KeccakStarkConfig(_pcs(1)), Sha256StarkConfig(_pcs(1))]
CONFIG_IDS = ["poseidon2", "keccak", "sha256"]


@pytest.mark.parametrize("config", CONFIGS, ids=CONFIG_IDS)
@pytest.mark.parametrize("air,message", [
    (KeccakAir(KoalaBear), "the Keccak AIR has no sharded quotient kernel"),
    (_poseidon2(BabyBear, 13), f"the Poseidon2 AIR over {BabyBear.name} has no sharded quotient kernel"),
    (PE.mul_fib_pair_air(KoalaBear, 8), "the AIR has 2 preprocessed columns"),
    (SymbolicAir(KoalaBear, 6, _fib), "a trace of 6 columns: .*multiples of 4 columns"),
    (object(), "object is not an air.SymbolicAir"),
], ids=["keccak-f", "poseidon2-babybear", "preprocessed", "width-6", "not-an-air"])
def test_refused_before_any_device_call(config, air, message):
    with pytest.raises(ValueError, match="CosetBlockedTrace: " + message):
        CosetBlockedTrace(Untouchable(), config, air)
    with pytest.raises(ValueError, match="CosetBlockedTrace: " + message):
        prove_coset_blocked(config, air, Untouchable())


def test_an_unknown_configuration_is_refused():
    with pytest.raises(ValueError, match="CosetBlockedTrace: object is not a StarkConfig or KeccakStarkConfig"):
        CosetBlockedTrace(Untouchable(), object(), Blake3Air(KoalaBear))


def test_a_trace_below_the_block_height_is_refused():
    shard = CosetBlockedTrace(Untouchable(), KeccakStarkConfig(_pcs(1)), SymbolicAir(KoalaBear, 8, _fib))
    with pytest.raises(ValueError, match="CosetBlockedTrace: a trace of 512 rows: .* at least 1024 rows"):
        shard.commit(Untouchable(), torch.zeros((512, 8), dtype=torch.int32))


@pytest.mark.parametrize("log_blowup", [2, 3])
def test_a_quotient_domain_smaller_than_the_lde_domain_is_refused(log_blowup):
    with pytest.raises(ValueError, match=f"log_num_quotient_chunks 1 .* differs from log_blowup {log_blowup}"):
        prove_coset_blocked(KeccakStarkConfig(_pcs(log_blowup)), Sha256Air(KoalaBear), Untouchable())


@pytest.mark.parametrize("config", CONFIGS, ids=CONFIG_IDS)
@pytest.mark.parametrize("air", [Blake3Air(BabyBear), Blake3Air(KoalaBear), Sha256Air(KoalaBear), _poseidon2(KoalaBear, 20),
                                 SymbolicAir(KoalaBear, 8, _fib)], ids=["blake3-bb", "blake3-kb", "sha256", "poseidon2-kb", "symbolic"])
def test_the_blocked_airs_are_accepted(config, air):
    assert coset_blocked_error(config, air) is None


def test_memory_plan_is_twice_the_trace_plus_the_allowance():
    air = Blake3Air(KoalaBear)
    N, W = 1 << 20, 9168
    trace = N * W * 4
    assert trace == 38_453_379_072
    allowance = coset_blocked_allowance_bytes(W, 20, 1)
    # every coset's sub-tree (2N - 1 digests of 32 bytes), a 128-column chunk of coefficients, 64 bytes per LDE row per coset
    assert allowance == 2 * (2 * N - 1) * 32 + N * 128 * 4 + 64 * (2 * N) * 2
    assert coset_blocked_memory_bytes(air, 20, 1) == 2 * trace + allowance
    usable = 85 * 10**9                                          # an H100 80 GB card
    assert trace + 2 * trace > usable > coset_blocked_memory_bytes(air, 20, 1)
    sha = Sha256Air(KoalaBear)
    assert 3 * (N * 7728 * 4) > usable > coset_blocked_memory_bytes(sha, 20, 1)
    # four cosets: still twice the trace, the allowance grows with the LDE
    assert coset_blocked_memory_bytes(sha, 10, 2) == 2 * (1024 * 7728 * 4) + coset_blocked_allowance_bytes(7728, 10, 2)
    assert coset_blocked_allowance_bytes(8, 4, 0) == (2 * 16 - 1) * 32 + 16 * 8 * 4 + 64 * 16


@pytest.mark.parametrize("log_n,log_blowup", [(4, 1), (6, 2), (5, 3), (3, 4)])
def test_each_block_of_rows_is_one_coset_holding_its_next_rows(log_n, log_blowup):
    N, B = 1 << log_n, 1 << log_blowup
    log_h = log_n + log_blowup
    for k in range(B):
        nat = _bitrev(np.arange(k * N, (k + 1) * N, dtype=np.int64), log_h)
        assert np.array_equal(nat, quotient_slice_natural_indices(k, N, log_h))
        # natural index i is the point g w_H^i: the block is the coset g w_H^bitrev(k) <w_N>, each point once
        assert np.all(nat % B == _bitrev(k, log_blowup))
        assert sorted((nat // B).tolist()) == list(range(N))
        # the next row of point i is i + B (w_N = w_H^B), which lies in the same coset
        assert next_row_rank(k, B, log_blowup) == k
        assert np.all(((nat + B) % (N * B)) % B == nat % B)


def test_natural_order_undoes_the_bit_reversed_block_slices():
    log_h = 7
    H = 1 << log_h
    q = torch.arange(H * 4, dtype=torch.int32).reshape(H, 4)
    nat = natural_order(q, log_h)
    idx = _bitrev(np.arange(H, dtype=np.int64), log_h)
    assert torch.equal(nat, q[torch.from_numpy(idx)])
    assert torch.equal(natural_order(nat, log_h), q)
