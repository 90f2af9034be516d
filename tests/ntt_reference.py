"""A plain reference for the DFT family and the coset LDE: a textbook radix-2 transform on canonical values in int64 torch
tensors, on whatever device its input lives on.

It shares no code with the kernels or the C oracle: no Montgomery arithmetic, Shoup constants or twiddle heaps.  Values
cross in and out in the library's Montgomery form (x * 2^32 mod p) and are converted at the edges; everything in between is
canonical, with every product (< 2^62) reduced by int64 `%`.  Twiddles are powers of the 2^k-th root
pow(TOP_ROOT, 2^(TWO_ADICITY - k), p), the first power by Python `pow` and the rest by doubling the list in torch.

The semantics are the reference's (dft/src/traits.rs), which oracle/p3_oracle.c restates:
  dft         y_i = sum_j x_j w^(ij), w the generator of the size-h subgroup, natural order in and out;
  idft        the inverse: dft with w^-1, divided by h;
  coset_dft   row i scaled by s^i, then dft (evaluations on s * H);
  coset_idft  idft, then row i scaled by s^-i;
  coset_lde   the evaluations of the interpolant of the (h, w) input on s * K, |K| = h << added_bits: idft, zero-pad to |K|
              rows, coset_dft over K.  Natural row i holds the point s * g^i; with bitrev_out, memory row r holds natural row
              bitrev(r) (the layout the LDE kernels write and TwoAdicFriPcs commits).

Wide matrices go through in column chunks of at most MAX_WORDS words of the largest intermediate, so that the peak memory of
a call stays bounded (a few times MAX_WORDS * 8 bytes) whatever the width."""
import torch

MAX_WORDS = 1 << 27     # int64 words per column chunk of the largest intermediate: 1 GiB


def column_chunks(rows, w, max_words=None):
    """Column ranges [c0, c1) of an (rows, w) matrix with at most max_words (default MAX_WORDS) words each (at least one
    column)."""
    step = max(1, (max_words or MAX_WORDS) // rows)
    return [(c0, min(w, c0 + step)) for c0 in range(0, w, step)]


def to_canonical(f, m):
    """Montgomery (int64 or int32 holding u32 words) -> canonical int64: x * 2^-32 mod p."""
    x = m.to(torch.int64) & 0xFFFFFFFF
    return x * pow(1 << 32, f.P - 2, f.P) % f.P


def to_monty(f, x):
    """Canonical int64 -> Montgomery int64: x * 2^32 mod p."""
    return (x << 32) % f.P


def _root(f, log_n):
    return pow(f.TOP_ROOT, 1 << (f.TWO_ADICITY - log_n), f.P)


def _powers(f, g, n, device):
    """g^0 .. g^(n-1) mod p (g canonical), as an int64 tensor."""
    pw = torch.ones(1, dtype=torch.int64, device=device)
    while pw.numel() < n:
        pw = torch.cat([pw, pw * pow(g, pw.numel(), f.P) % f.P])
    return pw[:n]


def _bitrev(log_n, device):
    i = torch.arange(1 << log_n, dtype=torch.int64, device=device)
    r = torch.zeros_like(i)
    for b in range(log_n):
        r |= ((i >> b) & 1) << (log_n - 1 - b)
    return r


def _log2(n):
    assert n > 0 and n & (n - 1) == 0, f"height {n} is not a power of two"
    return n.bit_length() - 1


def _ntt(f, x, g):
    """The size-n DFT of every column of x (canonical int64, (n, c)) with the primitive n-th root g: natural order in and
    out.  Iterative radix-2 DIT after a bit-reversal gather; returns a new tensor."""
    n, p = x.shape[0], f.P
    log_n = _log2(n)
    x = x[_bitrev(log_n, x.device)]
    tw = _powers(f, g, max(1, n // 2), x.device)
    half = 1
    while half < n:
        v = x.view(n // (2 * half), 2, half, -1)
        a, b = v[:, 0], v[:, 1]
        b.mul_(tw[::n // (2 * half)].view(half, 1)).remainder_(p)        # b * w_{2 half}^j
        t = a - b
        a.add_(b).remainder_(p)
        b.copy_(t.remainder_(p))
        del t
        half *= 2
    return x


def _scale_rows(f, x, s):
    """Row i of x times s^i (s canonical), in place."""
    x.mul_(_powers(f, s, x.shape[0], x.device).view(-1, 1)).remainder_(f.P)
    return x


def _chunked(rows_out, m, fn):
    """fn applied to m's column chunks (Montgomery int64 in and out), concatenated."""
    parts = [fn(m[:, c0:c1]) for c0, c1 in column_chunks(max(rows_out, m.shape[0]), m.shape[1])]
    return parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)


def _idft_canonical(f, x):
    n = x.shape[0]
    y = _ntt(f, x, pow(_root(f, _log2(n)), f.P - 2, f.P))
    return y.mul_(pow(n, f.P - 2, f.P)).remainder_(f.P)


def dft(f, m):
    return _chunked(m.shape[0], m, lambda c: to_monty(f, _ntt(f, to_canonical(f, c), _root(f, _log2(c.shape[0])))))


def idft(f, m):
    return _chunked(m.shape[0], m, lambda c: to_monty(f, _idft_canonical(f, to_canonical(f, c))))


def coset_dft(f, m, shift):
    """shift: Montgomery, as the library and the oracle take it."""
    s = f.from_monty(shift)
    return _chunked(m.shape[0], m, lambda c: to_monty(f, _ntt(f, _scale_rows(f, to_canonical(f, c), s), _root(f, _log2(c.shape[0])))))


def coset_idft(f, m, shift):
    s_inv = pow(f.from_monty(shift), f.P - 2, f.P)
    return _chunked(m.shape[0], m, lambda c: to_monty(f, _scale_rows(f, _idft_canonical(f, to_canonical(f, c)), s_inv)))


def coset_lde(f, m, added_bits, shift, bitrev_out=True):
    """(h, w) evaluations on H (Montgomery) -> (h << added_bits, w) evaluations on shift * K (Montgomery)."""
    h = m.shape[0]
    H = h << added_bits
    log_H = _log2(H)
    s = f.from_monty(shift)

    def one(c):
        coeffs = torch.zeros((H, c.shape[1]), dtype=torch.int64, device=c.device)
        coeffs[:h] = _idft_canonical(f, to_canonical(f, c))
        y = _ntt(f, _scale_rows(f, coeffs, s), _root(f, log_H))
        del coeffs
        if bitrev_out:
            y = y[_bitrev(log_H, y.device)]
        return to_monty(f, y)

    return _chunked(H, m, one)
