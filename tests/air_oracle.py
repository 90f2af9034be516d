"""Oracle of the constraint-program quotient (p3gpu_air_quotient_dev) — test infrastructure.

Evaluates an AIR's node DAG (include/p3gpu.h p3gpu_air_node) directly over the quotient domain with the reference's formulas, in
int64 torch tensors of canonical integers reduced with `%` (no Montgomery arithmetic, as tests/ntt_reference.py); it never goes
through the compiled program, so it is independent of the compiler:

    quotient domain   g * K, |K| = 2^log_q;  natural index i <-> memory row bitrev(i) of the committed bit-reversed LDE prefix
    next row          natural index (i + 2^q) mod |K|, q = log_q - log_n (vertically_packed_row wraps)
    selectors         selectors_on_coset (commit/src/domain.rs:321-361), unnormalised:
                      Z_H(x) = x^N - 1, first = Z_H / (x - 1), last = Z_H / (x - w_N^-1), transition = x - w_N^-1
    fold              sum_k c_k alpha^(K - 1 - k)  (decompose_alpha, air/src/symbolic/builder.rs:482-511)
    quotient          fold / Z_H(x)

It runs where its LDE lives: a torch tensor is evaluated on its own device and the quotient comes back as an int32 tensor of u32
words there; a numpy array is evaluated on the CPU and the quotient comes back as a uint32 array.  Natural indices go through in
chunks, each gathering its own local and next rows and computing its own selectors, sized so that at most about MAX_WORDS int64
words are live at once whatever the domain size and the number of live DAG values.
"""
import numpy as np
import torch

from ntt_reference import MAX_WORDS

CONST, MAIN_LOCAL, MAIN_NEXT, PUBLIC, IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION, ADD, SUB, NEG, MUL = range(11)

_PRIMES = {0: 0x78000001, 1: 0x7F000001}
_GEN = {0: 31, 1: 3}
_W = {0: 11, 1: 3}
_TOP = {0: (0x1A427A41, 27), 1: (0x6AC49F88, 24)}


def _root(fid, bits):
    top, adicity = _TOP[fid]
    return pow(top, 1 << (adicity - bits), _PRIMES[fid])


def _vpow(x, e, p):
    r = torch.ones_like(x)
    b = x.clone()
    while e:
        if e & 1:
            r = r * b % p
        b = b * b % p
        e >>= 1
    return r


def _powers(w, n, p, device):
    """w^0 .. w^(n-1) as int64 (doubling)."""
    out = torch.ones(n, dtype=torch.int64, device=device)
    k = 1
    while k < n:
        out[k:2 * k] = out[:min(k, n - k)] * pow(w, k, p) % p
        k *= 2
    return out


def _bitrev(i, n_bits):
    r = torch.zeros_like(i)
    for b in range(n_bits):
        r |= ((i >> b) & 1) << (n_bits - 1 - b)
    return r


def _ef_mul(a, b, p, w):
    r = [0] * 7
    for i in range(4):
        for j in range(4):
            r[i + j] += a[i] * b[j]
    return [(r[0] + w * r[4]) % p, (r[1] + w * r[5]) % p, (r[2] + w * r[6]) % p, r[3] % p]


def _schedule(nodes, cons):
    """Per node: how many later reads it has (operands and constraint positions), the constraint positions it fills, and the most
    values the evaluation holds at once (an upper bound: constants and public values are counted as vectors)."""
    uses = [0] * len(nodes)
    positions = {}
    for k, node in enumerate(cons):
        uses[node] += 1
        positions.setdefault(node, []).append(k)
    for op, a, b, _ in nodes:
        if op in (ADD, SUB, MUL):
            uses[a] += 1; uses[b] += 1
        elif op == NEG:
            uses[a] += 1
    left, live, peak = list(uses), 0, 0
    for i, (op, a, b, _) in enumerate(nodes):           # air_quotients' evaluation order, counting instead of computing
        if left[i] == 0:
            continue
        live += 1
        peak = max(peak, live)
        for j in ((a, b) if op in (ADD, SUB, MUL) else (a,) if op == NEG else ()):
            left[j] -= 1
            live -= left[j] == 0
        left[i] -= len(positions.get(i, ()))
        live -= left[i] == 0
    return uses, positions, peak


def air_quotient(fid, nodes, constraints, lde_bitrev, log_q, log_n, public_values_monty, alpha_monty, *, chunk_points=None):
    """(2^log_q, 4) Montgomery quotient values in natural order: uint32 numpy for a numpy LDE, an int32 tensor of u32 words on the
    LDE's device for a torch LDE.  lde_bitrev: the committed bit-reversed LDE (>= 2^log_q rows, Montgomery); public values and
    alpha: Montgomery words.  chunk_points: natural indices per chunk (default: as many as MAX_WORDS allows)."""
    return air_quotients(fid, nodes, constraints, lde_bitrev, log_q, log_n, public_values_monty, [alpha_monty], chunk_points=chunk_points)[0]


def air_quotients(fid, nodes, constraints, lde_bitrev, log_q, log_n, public_values_monty, alphas_monty, *, chunk_points=None):
    """air_quotient for several alphas over one evaluation of the DAG: a list with one quotient per alpha."""
    p = _PRIMES[fid]
    rinv = pow(1 << 32, p - 2, p)
    c = lambda m: int(m) * rinv % p
    nodes = np.asarray(nodes, dtype=np.int64).reshape(-1, 4).tolist()
    cons = [int(k) for k in np.asarray(constraints).ravel()]
    size, q = 1 << log_q, log_q - log_n
    as_numpy = not isinstance(lde_bitrev, torch.Tensor)
    lde = torch.from_numpy(np.ascontiguousarray(np.asarray(lde_bitrev, dtype=np.uint32)[:size]).view(np.int32)) if as_numpy else lde_bitrev
    assert lde.dim() == 2 and lde.shape[0] >= size, f"LDE of shape {tuple(lde.shape)}: need at least 2^{log_q} rows"
    dev = lde.device
    uses, positions, peak = _schedule(nodes, cons)
    n_alpha = len(alphas_monty)
    if chunk_points is None:
        chunk_points = max(1, MAX_WORDS // (peak + 4 * n_alpha + 16))

    K = len(cons)
    apow = []
    for al in alphas_monty:
        alpha = [c(v) for v in np.asarray(al).ravel()]
        pw = [[1, 0, 0, 0]]
        for _ in range(max(K - 1, 0)):
            pw.append(_ef_mul(pw[-1], alpha, p, _W[fid]))
        apow.append(pw)
    # ap[k]: (n_alpha, 1, 4), the factor of the constraint at position k
    ap = torch.tensor(apow, dtype=torch.int64, device=dev).reshape(n_alpha, max(K, 1), 4).permute(1, 0, 2).unsqueeze(2) if K else None

    g, w = _GEN[fid], _root(fid, log_q)
    w_inv = pow(_root(fid, log_n), p - 2, p)
    # Z_H(x) = g^N w^(i N) - 1 depends on i mod 2^q only
    zh_tab = [(pow(g, 1 << log_n, p) * pow(w, j << log_n, p) - 1) % p for j in range(1 << q)]
    zh_all = torch.tensor(zh_tab, dtype=torch.int64, device=dev)
    izh_all = torch.tensor([pow(z, p - 2, p) for z in zh_tab], dtype=torch.int64, device=dev)
    pubs = [c(v) for v in public_values_monty]

    out = torch.empty((n_alpha, size, 4), dtype=torch.int32, device=dev)
    for i0 in range(0, size, chunk_points):
        nat = torch.arange(i0, min(size, i0 + chunk_points), dtype=torch.int64, device=dev)
        n = nat.numel()
        rows = _bitrev(nat, log_q)
        nrows = None
        zh = zh_all[nat & ((1 << q) - 1)]
        selectors = {}

        def selector(op):
            if not selectors:
                x = _powers(w, n, p, dev) * (g * pow(w, i0, p) % p) % p
                selectors[IS_FIRST_ROW] = zh * _vpow((x - 1) % p, p - 2, p) % p
                selectors[IS_LAST_ROW] = zh * _vpow((x - w_inv) % p, p - 2, p) % p
                selectors[IS_TRANSITION] = (x - w_inv) % p
            return selectors[op]

        def column(r, col):
            return (lde[r, col].to(torch.int64) & 0xFFFFFFFF) * rinv % p

        left = list(uses)
        vals = {}

        def take(i):
            v = vals[i]
            left[i] -= 1
            if left[i] == 0:
                del vals[i]
            return v

        acc = torch.zeros((n_alpha, n, 4), dtype=torch.int64, device=dev)
        for i, (op, a, b, imm) in enumerate(nodes):
            if left[i] == 0:
                continue
            if op == CONST:
                v = c(imm)
            elif op == MAIN_LOCAL:
                v = column(rows, a)
            elif op == MAIN_NEXT:
                if nrows is None:
                    nrows = _bitrev((nat + (1 << q)) & (size - 1), log_q)
                v = column(nrows, a)
            elif op == PUBLIC:
                v = pubs[a]
            elif op in (IS_FIRST_ROW, IS_LAST_ROW, IS_TRANSITION):
                v = selector(op)
            elif op == ADD:
                v = (take(a) + take(b)) % p
            elif op == SUB:
                v = (take(a) - take(b)) % p
            elif op == NEG:
                v = (-take(a)) % p
            elif op == MUL:
                v = take(a) * take(b) % p
            else:
                raise ValueError(f"unknown op {op}")
            # constraints are folded as soon as their value exists (the sum's order does not matter): the value is dropped unless a
            # later node reads it
            for k in positions.get(i, ()):
                term = ap[K - 1 - k] * (v.view(1, n, 1) if isinstance(v, torch.Tensor) else v)
                acc += term % p
                left[i] -= 1
            if left[i]:
                vals[i] = v
        quo = acc % p * izh_all[nat & ((1 << q) - 1)].view(1, n, 1) % p
        out[:, i0:i0 + n] = ((quo << 32) % p).to(torch.int32)
    res = list(out.unbind(0))
    return [r.numpy().view(np.uint32) for r in res] if as_numpy else res
