"""tests/ntt_reference.py, the int64 transform the GPU tests check the large LDE and DFT shapes against, pinned on the CPU:
against the O(h^2) definition and against the C oracle for both fields, every transform kind, both row orders of the LDE and
several shifts.  Also the comparison the GPU tests report mismatches with (test_gpu_lde_paths._check_output), on CPU tensors."""
import numpy as np
import pytest
import torch

from oracle import p3_oracle as O
import ntt_reference as R
from test_gpu_lde_paths import G, POISON, _check_output

from plonky3_b200.field import BabyBear, KoalaBear

FIELDS = [BabyBear, KoalaBear]


def _t(m):
    return torch.from_numpy(m.astype(np.int64))


def _shifts(f):
    return {"one": f.ONE, "generator": f.generator, "random": int(O.random_matrix(f.id, 1, 1, seed=99 + f.id)[0, 0])}


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
def test_roots_match_oracle_at_full_two_adicity(f):
    # the comparisons below reach roots of order up to 2^17; the large GPU cases use them up to 2^TWO_ADICITY: every root order
    # against the oracle's own generators, so the reference does not rest on one shared constant
    for k in range(f.TWO_ADICITY + 1):
        assert f.to_monty(R._root(f, k)) == O.two_adic_generator(f.id, k), k
    g = R._root(f, f.TWO_ADICITY)
    assert pow(g, 1 << (f.TWO_ADICITY - 1), f.P) == f.P - 1     # primitive: order exactly 2^TWO_ADICITY


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h", range(6))
def test_dft_matches_definition(f, log_h):
    m = O.random_matrix(f.id, 1 << log_h, 3, seed=log_h)
    assert np.array_equal(R.dft(f, _t(m)).numpy(), O.naive_dft(f.id, m))


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h", range(15))
def test_dft_kinds_match_oracle(f, log_h):
    m = O.random_matrix(f.id, 1 << log_h, 3, seed=100 + log_h)
    x = _t(m)
    assert np.array_equal(R.dft(f, x).numpy(), O.dft_batch(f.id, m))
    assert np.array_equal(R.idft(f, x).numpy(), O.idft_batch(f.id, m))
    for name, s in _shifts(f).items():
        assert np.array_equal(R.coset_dft(f, x, s).numpy(), O.coset_dft_batch(f.id, m, s)), name
        assert np.array_equal(R.coset_idft(f, x, s).numpy(), O.coset_idft_batch(f.id, m, s)), name


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("log_h", range(15))
@pytest.mark.parametrize("added_bits", range(4))
def test_coset_lde_matches_oracle(f, log_h, added_bits):
    m = O.random_matrix(f.id, 1 << log_h, 2, seed=200 + 10 * log_h + added_bits)
    x = _t(m)
    for name, s in _shifts(f).items():
        for bitrev in (True, False):
            got = R.coset_lde(f, x, added_bits, s, bitrev_out=bitrev).numpy()
            assert np.array_equal(got, O.coset_lde_batch(f.id, m, added_bits, s, bitrev_out=bitrev)), (name, bitrev)


def test_column_chunks_match_whole_matrix():
    # a budget of 2^12 words splits a 2^9 x 21 LDE (2^10 rows out) into column chunks of 4, the last one ragged
    f = KoalaBear
    m = O.random_matrix(f.id, 1 << 9, 21, seed=5)
    assert R.column_chunks(1 << 10, 21, 1 << 12) == [(0, 4), (4, 8), (8, 12), (12, 16), (16, 20), (20, 21)]
    want = O.coset_lde_batch(f.id, m, 1, f.generator, bitrev_out=True)
    got = torch.cat([R.coset_lde(f, _t(m[:, c0:c1]), 1, f.generator) for c0, c1 in R.column_chunks(1 << 10, 21, 1 << 12)], dim=1)
    assert np.array_equal(got.numpy(), want)


def test_int32_words_convert_like_int64():
    # the device buffers hold u32 words as int32: canonical conversion must read them unsigned
    f = BabyBear
    w = torch.tensor([0, 1, f.P - 1, -1], dtype=torch.int32)
    assert R.to_canonical(f, w).tolist() == [f.from_monty(v) for v in (0, 1, f.P - 1, 0xFFFFFFFF)]
    assert R.to_monty(f, R.to_canonical(f, w[:3])).tolist() == [0, 1, f.P - 1]


# ------------------------------------------------------------------------------------------ the comparison
def _output(f, h, w, added_bits, off=0):
    """A (rows, w) reference LDE in a guarded int32 buffer at word G + off, as the GPU tests lay out a kernel's output."""
    m = O.random_matrix(f.id, h, w, seed=7)
    exp = R.coset_lde(f, _t(m), added_bits, f.generator)
    buf = torch.full((exp.numel() + 2 * G + off,), -1, dtype=torch.int32)
    buf[G + off:G + off + exp.numel()] = exp.view(-1).to(torch.int32)
    return buf, exp


def _where(row, col):
    return f"<row {row} col {col}>"


@pytest.mark.parametrize("as_oracle", [False, True])
def test_comparison_passes_the_reference(as_oracle):
    f = KoalaBear
    buf, exp = _output(f, 64, 5, 1, off=1)
    _check_output(f, buf, 1, 128, 5, exp.numpy().astype(np.uint32) if as_oracle else (lambda c0, c1: exp[:, c0:c1]), _where, "x")


@pytest.mark.parametrize("as_oracle", [False, True])
def test_comparison_reports_a_flipped_word(as_oracle):
    f = BabyBear
    buf, exp = _output(f, 64, 5, 2)
    buf[G + 77 * 5 + 3] ^= 1 << 7
    want = exp.numpy().astype(np.uint32) if as_oracle else (lambda c0, c1: exp[:, c0:c1])
    ref = "the oracle" if as_oracle else "the reference"
    with pytest.raises(pytest.fail.Exception, match=rf"1 of 1280 words in columns 0-4 differ from {ref}; first at row 77, column 3: .*<row 77 col 3>"):
        _check_output(f, buf, 0, 256, 5, want, _where, "x")


def test_comparison_reports_an_unwritten_word():
    f = KoalaBear
    buf, exp = _output(f, 32, 3, 0)
    buf[G + 31 * 3] = -1
    with pytest.raises(pytest.fail.Exception, match=r"not canonical; first at row 31, column 0: 0xffffffff \(the poison: never written\)"):
        _check_output(f, buf, 0, 32, 3, lambda c0, c1: exp[:, c0:c1], _where, "x")
    assert POISON == 0xFFFFFFFF


def test_comparison_reports_a_guard_word():
    f = KoalaBear
    buf, exp = _output(f, 32, 3, 0)
    buf[G + 96 + 2] = 5
    with pytest.raises(pytest.fail.Exception, match=r"wrote outside its output, 3 word\(s\) after it"):
        _check_output(f, buf, 0, 32, 3, lambda c0, c1: exp[:, c0:c1], _where, "x")


def test_comparison_reports_the_column_of_a_later_chunk(monkeypatch):
    # chunked comparison: a mismatch in the third column chunk is reported with its column in the whole matrix
    f = BabyBear
    buf, exp = _output(f, 16, 10, 0)
    monkeypatch.setattr(R, "MAX_WORDS", 48)
    buf[G + 9 * 10 + 7] = (int(exp[9, 7]) + 1) % f.P
    with pytest.raises(pytest.fail.Exception, match=r"1 of 48 words in columns 6-8 differ from the reference; first at row 9, column 7"):
        _check_output(f, buf, 0, 16, 10, lambda c0, c1: exp[:, c0:c1], _where, "x")
