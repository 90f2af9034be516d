"""Every coset-LDE and DFT kernel path of csrc/ntt.cu against the CPU oracle, on poisoned buffers.

`coset_lde_impl` picks one of several plans by height, width, pointer alignment, coset count and row order, and the fused
middle pass (`ntt_lde_mid_kernel`) has one kernel instance per tile width (`lde_mid_tile_width`: 16, 20 or a runtime 4-12).
Each case below pins one plan or instance, and asserts the launch count that identifies it, so a dispatch change that moves a
case off its path fails here instead of leaving the path unchecked:
  3 launches                 the fused path (inverse pass 1, ntt_lde_mid_kernel, forward pass 2);
  4 launches                 two-pass LDE with bit-reversed rows that the fused path refuses (four separate passes);
  2 + 2 * 2^added_bits       two-pass LDE in natural row order (one remapped forward network per coset).

run_lde_checked / run_dft_checked make a missing store visible.  The context keeps its scratch buffers between calls and torch's
caching allocator hands a freed block back to the next allocation of that size, so a second call on the same input would find
correct data from the first wherever it failed to write.  The helpers therefore run a dirty call on other data first, write the
result into a buffer filled with 0xFFFFFFFF (not canonical in either field) with guard words on both sides, and check the guards,
that every word is canonical, and the values; a failure names the coset and the row and column tiles it falls in.

A numpy input is checked against the CPU oracle.  Shapes too large for it take a DeviceInput (a seeded random matrix made on the
device) and are checked on the device, column chunk by column chunk, against tests/ntt_reference.py."""
import numpy as np
import pytest
import torch

from oracle import p3_oracle as O
import ntt_reference as R

from plonky3_b200 import _lib
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs, split_evals
from plonky3_b200.gpu import default_gpu

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]
G = 64                  # guard words on each side of an output
POISON = 0xFFFFFFFF     # >= p in both fields: a word no kernel wrote fails the canonical check


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert _lib.LIB_PATH.exists(), "libp3gpu.so missing — the CUDA path must be the one that runs"
    return default_gpu(0)


# ------------------------------------------------------------------------------------------ checked calls
def _brev(x, bits):
    return int(format(x, f"0{bits}b")[::-1], 2) if bits else 0


def _choose_tile_width(w):
    """csrc/ntt.cu choose_tile_width: column tile of the cp.async pass kernel."""
    if w <= 24:
        return w
    for ct in (16, 20, 24, 12):
        if w % ct == 0:
            return ct
    n = (w + 19) // 20
    return min(24, (-(-w // n) + 3) & ~3)


def _lde_mid_tile_width(w):
    """csrc/ntt.cu lde_mid_tile_width: column tile of the fused middle pass (0 = not fused)."""
    ct = _choose_tile_width(w)
    if w % 4 or ct % 4 or ct > 24:
        return 0
    return 12 if ct == 24 else ct


def _tiles(log_n, w, pos, col, fused):
    """The tiles that network position `pos` of a size-2^log_n network and column `col` fall in (two-pass plans)."""
    ct = _choose_tile_width(w)
    s = f"pass column tile {col // ct} ({ct}-column tiles)"
    if fused:
        fct = _lde_mid_tile_width(w)
        s += f", fused column tile {col // fct} ({fct}-column tiles)"
    if not 11 <= log_n <= 20:
        return s + f", network position {pos}"
    # plan_passes: layers [0, r1) then [r1, n), r1 = ceil(n / 2); a first-pass tile shares the low n - r1 bits of the position,
    # a last-pass tile the top r1 bits (the fused pass works on first-pass tiles)
    r2 = log_n // 2
    return s + f", first-pass row tile {pos & ((1 << r2) - 1)}, last-pass row tile {pos >> r2}"


class DeviceInput:
    """A uniform random (h, w) matrix of Montgomery words made on the device from a seed, for shapes too large for the CPU
    oracle: the checked calls fill their input buffer with it after the dirty call, and check the result against
    ntt_reference on the device."""

    def __init__(self, h, w, seed):
        self.shape, self.seed = (h, w), seed


def _fill_input(f, x, m):
    """x (flat int32 device buffer) <- m: a numpy matrix, or the DeviceInput's matrix drawn in place."""
    if isinstance(m, DeviceInput):
        x.random_(0, f.P, generator=torch.Generator(device=x.device).manual_seed(m.seed))
    else:
        x.copy_(torch.from_numpy(np.ascontiguousarray(m, dtype=np.uint32).view(np.int32).ravel()))


def _poisoned(words):
    return torch.full((words + 2 * G,), -1, dtype=torch.int32, device="cuda")


def check_matrix(f, got, exp, where, what, ref="the reference"):
    """got: an (rows, w) int32 tensor of u32 words on any device (a view is fine); exp(c0, c1): the expected columns [c0, c1) as
    an int64 tensor of Montgomery words on got's device.  Column chunk by column chunk (bounded memory), every word must be
    canonical and equal to exp; a failure names its row and column, the word, and where(row, col)."""
    rows, w = got.shape
    for c0, c1 in R.column_chunks(rows, w):
        g = got[:, c0:c1].to(torch.int64) & 0xFFFFFFFF
        want = exp(c0, c1)
        for label, bad in (("not canonical", g >= f.P), (f"differ from {ref}", g != want)):
            if bool(bad.any()):
                i = int(torch.argmax(bad.view(-1).to(torch.uint8)))
                row, col = divmod(i, c1 - c0)
                val = int(g[row, col])
                note = " (the poison: never written)" if val == POISON else ""
                pytest.fail(f"{what}: {int(bad.sum())} of {rows * (c1 - c0)} words in columns {c0}-{c1 - 1} {label}; first at row "
                            f"{row}, column {c0 + col}: 0x{val:08x}{note}, expected 0x{int(want[row, col]):08x}; {where(row, c0 + col)}")
        del g, want


def _check_output(f, buf, off, rows, w, exp, where, what):
    """buf: the whole flat output buffer (int32 tensor), the (rows, w) result at word G + off; exp: the expected matrix, a numpy
    array (the oracle's) or a function of a column range as check_matrix takes it (the reference's)."""
    n = rows * w
    lo, hi = buf[:G + off], buf[G + off + n:]
    for side, guard in (("before", lo.flip(0)), ("after", hi)):
        bad = guard != -1
        if bool(bad.any()):
            k = int(torch.argmax(bad.to(torch.uint8)))
            pytest.fail(f"{what}: wrote outside its output, {k + 1} word(s) {side} it "
                        f"(0x{int(guard[k]) & 0xFFFFFFFF:08x}; {int(bad.sum())} guard words changed)")
    ref = "the reference"
    if isinstance(exp, np.ndarray):
        e, ref = exp, "the oracle"
        exp = lambda c0, c1: torch.from_numpy(e[:, c0:c1].astype(np.int64)).to(buf.device)
    check_matrix(f, buf[G + off:G + off + n].view(rows, w), exp, where, what, ref)


def _lde_dev(gpu, f, x, in_off, out, out_off, h, w, added_bits, shift, bitrev_rows):
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_coset_lde_batch_dev(gpu.h, f.id, x.data_ptr() + 4 * in_off, h, w, added_bits, shift,
                                               out.data_ptr() + 4 * (G + out_off), int(bitrev_rows)))


def run_lde_checked(gpu, f, m, added_bits, shift, bitrev_rows=True, in_off=0, out_off=0, launches=None):
    """p3gpu_coset_lde_batch_dev on m (Montgomery, (h, w): a numpy matrix or a DeviceInput) with the input at word offset in_off
    and the output at word offset out_off of poisoned, guarded buffers, after a dirty call on other data; checks the launch count
    (if given), the guards, that every word is canonical and the result against the oracle (numpy input) or ntt_reference
    (DeviceInput).  Returns the (h << added_bits, w) output as numpy for a numpy input."""
    h, w = m.shape
    log_h, H = h.bit_length() - 1, h << added_bits
    x, out = torch.empty(h * w + in_off, dtype=torch.int32, device="cuda"), _poisoned(H * w)
    x.random_(0, f.P, generator=torch.Generator(device="cuda").manual_seed(h * w + added_bits))
    _lde_dev(gpu, f, x, in_off, out, out_off, h, w, added_bits, shift, bitrev_rows)   # also builds the twiddle heaps
    _fill_input(f, x[in_off:], m)
    out.fill_(-1)
    n0 = gpu.launches
    _lde_dev(gpu, f, x, in_off, out, out_off, h, w, added_bits, shift, bitrev_rows)
    n = gpu.launches - n0
    what = f"{f.name} LDE 2^{log_h} x {w}, added_bits {added_bits}, {'bit-reversed' if bitrev_rows else 'natural'} rows"
    if launches is not None:
        assert n == launches, f"{what}: {n} launches instead of {launches}: the case left the path it pins"

    def where(row, col):
        if bitrev_rows:
            cb, pos = row >> log_h, row & (h - 1)
        else:
            cb, pos = _brev(row & ((1 << added_bits) - 1), added_bits), _brev(row >> added_bits, log_h)
        return f"coset {_brev(cb, added_bits)} (block {cb}), " + _tiles(log_h, w, pos, col, n == 3)

    if isinstance(m, DeviceInput):
        xm = x[in_off:].view(h, w)
        _check_output(f, out, out_off, H, w, lambda c0, c1: R.coset_lde(f, xm[:, c0:c1], added_bits, shift, bitrev_rows), where, what)
        return None
    _check_output(f, out, out_off, H, w, O.coset_lde_batch(f.id, m, added_bits, shift, bitrev_out=bitrev_rows), where, what)
    return out[G + out_off:G + out_off + H * w].cpu().numpy().view(np.uint32).reshape(H, w)


_ORACLE_DFT = {_lib.DFT: lambda f, m, s: O.dft_batch(f.id, m), _lib.IDFT: lambda f, m, s: O.idft_batch(f.id, m),
               _lib.COSET_DFT: lambda f, m, s: O.coset_dft_batch(f.id, m, s),
               _lib.COSET_IDFT: lambda f, m, s: O.coset_idft_batch(f.id, m, s)}
_KIND_NAME = {_lib.DFT: "DFT", _lib.IDFT: "iDFT", _lib.COSET_DFT: "coset DFT", _lib.COSET_IDFT: "coset iDFT"}


def _dft_dev(gpu, f, kind, x, in_off, out, out_off, h, w, shift):
    gpu._use_torch_stream()
    _lib.check(gpu.L.p3gpu_dft_batch_dev(gpu.h, f.id, kind, x.data_ptr() + 4 * in_off, out.data_ptr() + 4 * (G + out_off), h, w, shift))


_REFERENCE_DFT = {_lib.DFT: lambda f, m, s: R.dft(f, m), _lib.IDFT: lambda f, m, s: R.idft(f, m),
                  _lib.COSET_DFT: R.coset_dft, _lib.COSET_IDFT: R.coset_idft}


def run_dft_checked(gpu, f, kind, m, shift=0, in_off=0, out_off=0, launches=None):
    """p3gpu_dft_batch_dev, checked the way run_lde_checked checks the LDE.  Returns the (h, w) output as numpy for a numpy
    input."""
    h, w = m.shape
    log_h = h.bit_length() - 1
    x, out = torch.empty(h * w + in_off, dtype=torch.int32, device="cuda"), _poisoned(h * w)
    x.random_(0, f.P, generator=torch.Generator(device="cuda").manual_seed(h * w + kind))
    _dft_dev(gpu, f, kind, x, in_off, out, out_off, h, w, shift)
    _fill_input(f, x[in_off:], m)
    out.fill_(-1)
    n0 = gpu.launches
    _dft_dev(gpu, f, kind, x, in_off, out, out_off, h, w, shift)
    n = gpu.launches - n0
    what = f"{f.name} {_KIND_NAME[kind]} 2^{log_h} x {w}"
    if launches is not None:
        assert n == launches, f"{what}: {n} launches instead of {launches}: the case left the path it pins"
    # natural-order output: row k is network position bitrev(k), written by the remapped last pass
    where = lambda row, col: _tiles(log_h, w, _brev(row, log_h), col, False)
    if isinstance(m, DeviceInput):
        xm = x[in_off:].view(h, w)
        _check_output(f, out, out_off, h, w, lambda c0, c1: _REFERENCE_DFT[kind](f, xm[:, c0:c1], shift), where, what)
        return None
    _check_output(f, out, out_off, h, w, _ORACLE_DFT[kind](f, m, shift), where, what)
    return out[G + out_off:G + out_off + h * w].cpu().numpy().view(np.uint32).reshape(h, w)


# ------------------------------------------------------------------------------------------ from the definition
def _powmod(x, e, p):
    r, b = np.ones_like(x), x % p
    while e:
        if e & 1:
            r = r * b % p
        b, e = b * b % p, e >> 1
    return r


def _eval_from_definition(f, m, xs):
    """Values at the canonical points xs of the polynomials of degree < n that take the values m (Montgomery, natural order,
    (n, w)) on H = <w_n>: barycentric f(x) = (x^n - 1) / n * sum_i y_i w^i / (x - w^i), and y_k at x = w^k.  Canonical int64
    arithmetic with every product reduced before it is summed (< 2^62 each, sums of 2^16 terms < 2^47)."""
    p, n = f.P, m.shape[0]
    omega = pow(f.TOP_ROOT, 1 << (f.TWO_ADICITY - (n.bit_length() - 1)), p)
    wi = np.ones(1, dtype=np.int64)
    while wi.size < n:
        wi = np.concatenate([wi, wi * pow(omega, wi.size, p) % p])
    xs = np.asarray(xs, dtype=np.int64)
    d = (xs[:, None] - wi[None, :]) % p
    d[d == 0] = 1                               # points of H: read off below
    wt = wi[None, :] * _powmod(d, p - 2, p) % p
    acc = np.zeros((xs.size, m.shape[1]), dtype=np.int64)
    for r0 in range(0, n, 1 << 16):
        y = f.from_monty_array(m[r0:r0 + (1 << 16)]).astype(np.int64)
        for k in range(xs.size):
            acc[k] = (acc[k] + (y * wt[k, r0:r0 + (1 << 16), None] % p).sum(axis=0)) % p
    ninv = pow(n, p - 2, p)
    out = np.array([acc[k] * ((pow(int(x), n, p) - 1) * ninv % p) % p for k, x in enumerate(xs)], dtype=np.int64)
    for k, x in enumerate(xs):
        on_h = np.flatnonzero(wi == x)
        if on_h.size:
            out[k] = f.from_monty_array(m[on_h[0]]).astype(np.int64)
    return out


def check_rows_from_definition(f, m, lde, added_bits, shift, n_rows=4, seed=0):
    """n_rows rows of a bit-reversed LDE against the definition: memory row r holds the evaluation at shift * g^bitrev(r),
    g the generator of the 2^(log h + added_bits) subgroup.  Independent of the oracle's Montgomery code."""
    H = lde.shape[0]
    log_H = H.bit_length() - 1
    rows = [0, H - 1] + [int(r) for r in np.random.default_rng(seed).integers(1, H - 1, n_rows - 2)]
    g = pow(f.TOP_ROOT, 1 << (f.TWO_ADICITY - log_H), f.P)
    s = f.from_monty(shift)
    xs = [s * pow(g, _brev(r, log_H), f.P) % f.P for r in rows]
    want = _eval_from_definition(f, m, xs)
    got = f.from_monty_array(lde[rows]).astype(np.int64)
    for k, r in enumerate(rows):
        assert np.array_equal(got[k], want[k]), f"row {r} (point {xs[k]}) differs from the definition"


# ------------------------------------------------------------------------------------------ the fused path
# Width -> the ntt_lde_mid_kernel instance and tiles it pins (lde_mid_tile_width; the outer passes tile by choose_tile_width):
FUSED_WIDTHS = [
    4,    # runtime-width instance (CT_T = 0) at ct = 4: one tile, 16-byte TMA boxes (the config-5 quotient chunk's width)
    12,   # runtime-width instance, one 12-column tile
    20,   # CT_T = 20, one full tile
    36,   # runtime-width instance, three 12-column tiles (choose_tile_width picks 12)
    52,   # CT_T = 20, ragged last tile: 20 + 20 + 12 (the TMA store clips columns 52-59)
    56,   # CT_T = 20, ragged last tile: 20 + 20 + 16
    68,   # CT_T = 20, ragged last tile: 20 + 20 + 20 + 8
    72,   # 24-column pass tiles (3) beside 12-column fused tiles (6, runtime-width instance)
]


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", FUSED_WIDTHS)
@pytest.mark.parametrize("log_h,added_bits", [(14, 0), (14, 1), (14, 2), (18, 0), (18, 1), (18, 2), (20, 1)])
def test_fused_lde_tile_widths(gpu, f, w, log_h, added_bits, monkeypatch):
    # 2^14 (7 + 7 layers) and 2^18 (9 + 9) take the fused path only on the cp.async kernel (P3GPU_NTT_PIPE=0); 2^20 (10 + 10)
    # takes it by default.  At 2^20 four rows per case are also checked against the definition.
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    m = O.random_matrix(f.id, 1 << log_h, w, seed=20000 + 1000 * log_h + 10 * w + added_bits)
    lde = run_lde_checked(gpu, f, m, added_bits, f.generator, launches=3)
    if log_h == 20:
        check_rows_from_definition(f, m, lde, added_bits, f.generator, seed=w)


# ------------------------------------------------------------------------------------------ config-5 quotient
@pytest.mark.parametrize("chunk", [0, 1])
def test_quotient_chunk_lde_config5_shape(gpu, chunk):
    # commit_quotient in config 5 splits the 2^21 x 4 quotient (EF4, flattened) into two 2^20 x 4 chunks and LDEs chunk i with
    # blowup 2 and shift h^-i, h the 2^21 root: shift ONE for chunk 0.  Fused path, runtime-width instance at ct = 4.
    f = KoalaBear
    shift = f.inv(f.pow(f.two_adic_generator(21), chunk))
    m = O.random_matrix(f.id, 1 << 20, 4, seed=500 + chunk)
    lde = run_lde_checked(gpu, f, m, 1, shift, launches=3)
    check_rows_from_definition(f, m, lde, 1, shift, seed=chunk)


def test_quotient_ldes_config5_end_to_end(gpu):
    # TwoAdicFriPcs.get_quotient_ldes as commit_quotient calls it on the config-5 quotient (2^21 x 4 over GENERATOR * K, two
    # chunks), against the oracle LDE of each chunk; both chunk LDEs take the fused path.
    f = KoalaBear
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), None, FriParameters.new_benchmark_high_arity(None))
    log_n, chunks = 21, 2
    h = f.two_adic_generator(log_n)

    def evaluations(q):
        subs = split_evals(chunks, torch.from_numpy(q.view(np.int32)).cuda())
        return [((f.mul(f.generator, f.pow(h, i)), log_n - 1), s) for i, s in enumerate(subs)]

    pcs.get_quotient_ldes(evaluations(O.random_matrix(f.id, 1 << log_n, 4, seed=6)))   # twiddle heaps of both shifts
    q = O.random_matrix(f.id, 1 << log_n, 4, seed=5)
    n0 = gpu.launches
    ldes = pcs.get_quotient_ldes(evaluations(q))
    assert gpu.launches - n0 == 3 * chunks
    oh = O.two_adic_generator(f.id, log_n)
    for i, lde in enumerate(ldes):
        sub = np.ascontiguousarray(q[i::chunks])
        dshift = O.mul(f.id, f.generator, O.fpow(f.id, oh, i))
        exp = O.coset_lde_batch(f.id, sub, 1, O.mul(f.id, f.generator, O.inv(f.id, dshift)), bitrev_out=True)
        assert np.array_equal(lde.cpu().numpy().view(np.uint32), exp), f"chunk {i}"


# ------------------------------------------------------------------------------------------ fallbacks at two-pass heights
@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [100, 16])
@pytest.mark.parametrize("log_h", [16, 20])
@pytest.mark.parametrize("in_off,out_off", [(1, 0), (0, 1), (1, 1)])
def test_misaligned_pointers(gpu, f, w, log_h, in_off, out_off, monkeypatch):
    # a buffer that is not 16-byte aligned: the fused path is refused and the cp.async kernel runs its four passes with 4-byte
    # copies (vec16 = false) although w % 4 == 0
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    m = O.random_matrix(f.id, 1 << log_h, w, seed=30000 + 1000 * log_h + 10 * w + 2 * in_off + out_off)
    run_lde_checked(gpu, f, m, 1, f.generator, in_off=in_off, out_off=out_off, launches=4)


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [100, 16, 4])
@pytest.mark.parametrize("log_h", [14, 18, 20])
def test_eight_cosets(gpu, f, w, log_h, monkeypatch):
    # added_bits = 3: more than the fused pass's 4 cosets, so four launches, the last two over all 8 cosets' blocks
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    m = O.random_matrix(f.id, 1 << log_h, w, seed=40000 + 1000 * log_h + w)
    run_lde_checked(gpu, f, m, 3, f.generator, launches=4)


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [100, 20, 4])
@pytest.mark.parametrize("log_h", [18, 20])
@pytest.mark.parametrize("added_bits", [1, 2])
def test_natural_order_rows(gpu, f, w, log_h, added_bits, monkeypatch):
    # bitrev_rows = 0: one forward network per coset whose last pass writes network position i to natural row
    # (bitrev(i) << added_bits) + coset (9- and 10-layer remaps), with the intermediate in the second scratch buffer
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    m = O.random_matrix(f.id, 1 << log_h, w, seed=50000 + 1000 * log_h + 10 * w + added_bits)
    run_lde_checked(gpu, f, m, added_bits, f.generator, bitrev_rows=False, launches=2 + 2 * (1 << added_bits))


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [1, 6])
def test_full_height_without_16_byte_rows(gpu, f, w):
    # w % 4 != 0 at 2^20: no fused pass, four launches of the cp.async kernel with 4-byte copies (a 1- and a 6-column tile)
    m = O.random_matrix(f.id, 1 << 20, w, seed=60000 + w)
    run_lde_checked(gpu, f, m, 1, f.generator, launches=4)


# ------------------------------------------------------------------------------------------ extreme values
def _extreme(f, kind, h, w):
    m = np.zeros((h, w), dtype=np.uint32)
    if kind == "all_max":
        m[:] = f.P - 1
    elif kind == "one_column_max":
        m[:, w - 1] = f.P - 1
    else:
        m[1::2] = f.P - 1
    return m


@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("w", [20, 100])
@pytest.mark.parametrize("log_h", [16, 20])
@pytest.mark.parametrize("kind", ["all_max", "one_column_max", "alternating_rows"])
def test_fused_lde_extreme_inputs(gpu, f, w, log_h, kind, monkeypatch):
    # the largest canonical word (p - 1) everywhere, in one column, or on every other row: the lazy [0, 2p) values the fused
    # path carries between its passes and the final reduction of forward pass 2 at their extremes
    if log_h < 20:
        monkeypatch.setenv("P3GPU_NTT_PIPE", "0")
    run_lde_checked(gpu, f, _extreme(f, kind, 1 << log_h, w), 1, f.generator, launches=3)


# ------------------------------------------------------------------------------------------ DFT kinds
@pytest.mark.parametrize("f", FIELDS, ids=lambda f: f.name)
@pytest.mark.parametrize("kind", [_lib.DFT, _lib.IDFT, _lib.COSET_DFT, _lib.COSET_IDFT], ids=lambda k: _KIND_NAME[k].replace(" ", "_"))
@pytest.mark.parametrize("log_h", [18, 20])
@pytest.mark.parametrize("w", [4, 20, 52, 100])
def test_dft_kinds_two_pass(gpu, f, kind, log_h, w):
    # 9 + 9 layers (TMA pipeline for w >= 8, the cp.async kernel for w = 4) and 10 + 10 (cp.async kernel); the last pass
    # writes natural order through the bit-reversal remap.  The coset iDFT adds one row-scaling launch.
    m = O.random_matrix(f.id, 1 << log_h, w, seed=70000 + 1000 * log_h + 10 * w + kind)
    shift = f.to_monty(0x2345678 + log_h)
    run_dft_checked(gpu, f, kind, m, shift, launches=3 if kind == _lib.COSET_IDFT else 2)
