"""uni-stark `verify` for proofs in the reference's wire form (proof_io.py), mirroring

    uni-stark/src/verifier.rs:282-561   verify_with_preprocessed (non-ZK; preprocessed and periodic columns)
    fri/src/two_adic_pcs.rs:684-715     TwoAdicFriPcs::verify
    fri/src/verifier.rs:158-436         verify_fri;  :471-606 fold_query;  :617-833 open_inputs
    fri/src/two_adic_pcs.rs:108-131     TwoAdicFriFolding::fold_row

As in the reference, the verifier's arithmetic is scalar host code over a few thousand extension-field values (here on canonical
Python integers); what is batched is the hashing: every input batch and every FRI round is ONE amortised multi-opening check
(`Mmcs::verify_multi_batch`, merkle-tree/src/mmcs/mod.rs:430-), whose leaf hashes and per-level compressions go to the device through
the configuration's MMCS (merkle_tree.MerkleTreeMmcs.hash_rows / compress_pairs — one launch per tree level for all queries).  The
transcript is the configuration's challenger.  Nothing here knows how hashing is done: the CPU tests drive the same code with
oracle-backed stand-ins for the MMCS and the challenger (tests/stark_verify.py), which pins it on the reference's own committed proof.
"""
from __future__ import annotations

import numpy as np

from .merkle_tree import MerkleTreeError
from .proof_io import proof_from_postcard


class VerificationError(Exception):
    """uni-stark/src/verifier.rs VerificationError / fri/src/verifier.rs FriError, as one exception with the variant's message."""


def _need(cond, msg):
    if not cond:
        raise VerificationError(msg)


def _rev(i: int, bits: int) -> int:
    return int(format(i, "0%db" % bits)[::-1], 2) if bits else 0


class Ext:
    """F and F[X]/(X^4 - W) on canonical integers for one plonky3_b200.field.Field."""

    def __init__(self, field):
        self.field, self.P, self.W = field, field.P, field.EXT_W
        self.GEN = field.GENERATOR
        self.two_adicity = field.TWO_ADICITY

    def c(self, m): return self.field.from_monty(int(m))
    def m(self, x): return self.field.to_monty(int(x))
    def inv(self, x): return pow(x % self.P, self.P - 2, self.P)
    def root(self, bits): return self.field.from_monty(self.field.two_adic_generator(bits))
    def ec(self, words): return [self.c(v) for v in words]

    def mul(self, a, b):
        r = [0] * 7
        for i in range(4):
            for j in range(4):
                r[i + j] += a[i] * b[j]
        return [(r[0] + self.W * r[4]) % self.P, (r[1] + self.W * r[5]) % self.P, (r[2] + self.W * r[6]) % self.P, r[3] % self.P]

    def add(self, a, b): return [(x + y) % self.P for x, y in zip(a, b)]
    def sub(self, a, b): return [(x - y) % self.P for x, y in zip(a, b)]
    def scale(self, a, s): return [x * s % self.P for x in a]
    def base(self, x): return [x % self.P, 0, 0, 0]
    ONE = [1, 0, 0, 0]
    ZERO = [0, 0, 0, 0]

    def pow(self, a, e):
        r = [1, 0, 0, 0]
        while e:
            if e & 1:
                r = self.mul(r, a)
            a = self.mul(a, a); e >>= 1
        return r

    def inverse(self, a):
        """through the Frobenius conjugates (X -> zeta X, zeta = W^((p-1)/4)): a^-1 = conj1 conj2 conj3 / Norm(a)."""
        zeta = pow(self.W, (self.P - 1) // 4, self.P)
        conj = lambda k: [a[i] * pow(zeta, i * k, self.P) % self.P for i in range(4)]
        b = self.mul(self.mul(conj(1), conj(2)), conj(3))
        n = self.mul(a, b)
        _need(n[1] == n[2] == n[3] == 0 and n[0] != 0, "division by zero")
        return self.scale(b, self.inv(n[0]))

    def from_basis(self, coeffs):
        """from_ext_basis_coefficients: sum_k X^k * coeffs[k] (X * (a0..a3) = (W a3, a0, a1, a2))."""
        acc = [0, 0, 0, 0]
        for k, v in enumerate(coeffs):
            for _ in range(k):
                v = [self.W * v[3] % self.P, v[0], v[1], v[2]]
            acc = self.add(acc, v)
        return acc


def fold_row(e: Ext, index: int, log_height: int, log_arity: int, beta, evals):
    """two_adic_pcs.rs:108-131: the arity evaluations sit on the coset subgroup_start * <w_arity> (bit-reversed); interpolate, evaluate
    at beta."""
    arity = 1 << log_arity
    start = pow(e.root(log_height + log_arity), _rev(index, log_height), e.P)
    w = e.root(log_arity)
    xs = [start * pow(w, k, e.P) % e.P for k in range(arity)]
    xs = [xs[_rev(k, log_arity)] for k in range(arity)]
    acc = [0, 0, 0, 0]
    for j in range(arity):
        num, den = [1, 0, 0, 0], 1
        for k in range(arity):
            if k != j:
                num = e.mul(num, e.sub(beta, e.base(xs[k])))
                den = den * (xs[j] - xs[k]) % e.P
        acc = e.add(acc, e.mul(evals[j], e.scale(num, e.inv(den))))
    return acc


def _observe_cap(challenger, cap):
    """Observe a commitment as digests, not as field elements: a byte transcript (SerializingChallenger32 over a Keccak or SHA-256
    MMCS) absorbs a [u64; 4] or [u8; 32] digest as its 32 bytes, which the words' canonical values are not.  A transcript without observe_cap only ever sees
    [F; 8] digests, which are field elements."""
    getattr(challenger, "observe_cap", challenger.observe_slice)(np.asarray(cap, dtype=np.uint32))


def _check_witness(challenger, e: Ext, bits: int, witness_word: int) -> bool:
    """GrindingChallenger::check_witness (grinding_challenger.rs:60-70)."""
    if bits == 0:
        return True
    challenger.observe(int(witness_word))
    return challenger.sample_bits(bits) == 0


def verify_fri(e: Ext, params, input_mmcs, proof: dict, challenger, rounds):
    """fri/src/verifier.rs:158-436.  `rounds`: [(commitment, [(log_domain_size, [(z, values_at_z)])])], canonical EF lists."""
    _need(params.num_queries > 0, "FRI instance has zero queries")
    alpha = e.ec(challenger.sample_algebra_element())
    cpo = proof["commit_phase_openings"]
    _need(len(cpo) == len(proof["commit_phase_commits"]), "commit phase opening count mismatch")
    log_arities = []
    for r, o in enumerate(cpo):
        _need(1 <= o["log_arity"] <= params.max_log_arity, f"round {r}: invalid log-arity")
        _need(len(o["sibling_values"]) == params.num_queries, f"round {r}: opened query count mismatch")
        _need(all(len(s) == (1 << o["log_arity"]) - 1 for s in o["sibling_values"]), f"round {r}: sibling values length mismatch")
        log_arities.append(o["log_arity"])
    log_final_height = params.log_blowup + params.log_final_poly_len
    log_max = sum(log_arities) + log_final_height
    _need(log_max <= e.two_adicity, "global max height exceeds the field two-adicity")
    _need(max(ld + params.log_blowup for _, mats in rounds for ld, _ in mats) == log_max, "global max height mismatch")
    _need(len(proof["commit_pow_witnesses"]) == len(proof["commit_phase_commits"]), "commit PoW witness count mismatch")
    betas = []
    for cap, wit in zip(proof["commit_phase_commits"], proof["commit_pow_witnesses"]):
        _observe_cap(challenger, cap)
        _need(_check_witness(challenger, e, params.commit_proof_of_work_bits, wit), "invalid proof-of-work witness")
        betas.append(e.ec(challenger.sample_algebra_element()))
    final_poly = [e.ec(co) for co in proof["final_poly"]]
    _need(len(final_poly) == 1 << params.log_final_poly_len, "final polynomial length mismatch")
    challenger.observe_slice(np.asarray(proof["final_poly"], dtype=np.uint32))
    for la in log_arities:
        challenger.observe_canonical(la)
    _need(_check_witness(challenger, e, params.query_proof_of_work_bits, proof["query_pow_witness"]), "invalid proof-of-work witness")
    indices = [challenger.sample_bits(log_max) for _ in range(params.num_queries)]

    # open_inputs: one amortised check per batch, then the reduced openings per height
    io = proof["input_openings"]
    _need(len(io) == len(rounds), "input proof batch count mismatch")
    for b, (cap, mats) in zip(io, rounds):
        _need(len(b["opened_values"]) == len(indices), "opened query count mismatch")
        _need(all(len(ov) == len(mats) for ov in b["opened_values"]), "opened-values matrix count mismatch")
        _need(all(len(pts) > 0 for _, pts in mats), "matrix opened at no points")
        dims = [(len(pts[0][1]), 1 << (ld + params.log_blowup)) for ld, pts in mats]
        lh = max(h for _, h in dims).bit_length() - 1
        try:
            input_mmcs.verify_multi_batch(cap, dims, [i >> (log_max - lh) for i in indices], b["opened_values"], b["proof"])
        except MerkleTreeError as ex:
            raise VerificationError(f"input error: {ex}") from None
    reduced = []
    for q, index in enumerate(indices):
        ro = {}
        for b, (_, mats) in zip(io, rounds):
            for row, (ld, pts) in zip(b["opened_values"][q], mats):
                lh = ld + params.log_blowup
                x = e.GEN * pow(e.root(lh), _rev(index >> (log_max - lh), lh), e.P) % e.P
                apow, acc = ro.get(lh, (e.ONE, e.ZERO))
                px = e.ec(row)
                for z, ys in pts:
                    _need(len(ys) == len(px), "evaluation count mismatch")
                    den = e.sub(z, e.base(x))
                    _need(any(den), "query point coincides with the opening point")
                    quot = e.inverse(den)
                    for p_at_x, p_at_z in zip(px, ys):
                        acc = e.add(acc, e.mul(e.mul(apow, e.sub(p_at_z, e.base(p_at_x))), quot))
                        apow = e.mul(apow, alpha)
                ro[lh] = (apow, acc)
        if params.log_blowup in ro:
            _need(not any(ro[params.log_blowup][1]), "final polynomial mismatch")
        reduced.append(sorted(((lh, v[1]) for lh, v in ro.items()), reverse=True))

    # fold_query for every query; the reconstructed rows are authenticated afterwards, one check per round
    groups = [[] for _ in cpo]
    rows_by_round = [[] for _ in cpo]
    for q, (index, ro) in enumerate(zip(indices, reduced)):
        _need(ro and ro[0][0] == log_max, "missing initial reduced opening")
        ro = list(ro)
        folded = ro.pop(0)[1]
        cur, idx = log_max, index
        for r, (beta, la, o) in enumerate(zip(betas, log_arities, cpo)):
            arity = 1 << la
            pos = idx % arity
            sib = [e.ec(v) for v in o["sibling_values"][q]]
            evals = sib[:pos] + [folded] + sib[pos:]
            cur -= la
            idx >>= la
            folded = fold_row(e, idx, cur, la, beta, evals)
            groups[r].append(idx)
            rows_by_round[r].append([np.array([e.m(v) for ev in evals for v in ev], dtype=np.uint32)])
            if ro and ro[0][0] == cur:
                folded = e.add(folded, e.mul(e.pow(beta, arity), ro.pop(0)[1]))
        _need(cur == log_final_height, "final folded height mismatch")
        _need(not ro, "unconsumed reduced openings remain after folding")
        x = pow(e.root(log_max), _rev(idx, log_max), e.P)
        ev = [0, 0, 0, 0]
        for co in reversed(final_poly):
            ev = e.add(e.scale(ev, x), co)
        _need(ev == folded, "final polynomial mismatch")
    cur = log_max
    for r, (cap, o, la) in enumerate(zip(proof["commit_phase_commits"], cpo, log_arities)):
        cur -= la
        try:
            params.mmcs.verify_multi_batch(cap, [(4 << la, 1 << cur)], groups[r], rows_by_round[r], o["proof"])
        except MerkleTreeError as ex:
            raise VerificationError(f"commit phase MMCS error: {ex}") from None


def eval_periodic_poly(e: Ext, values, point):
    """fri/src/periodic.rs:209-259: the degree < p interpolant of `values` (canonical) over the subgroup of size p = len(values),
    at the EF point, by the barycentric form (x^p - 1) / p * sum_i v_i w^i / (x - w^i)."""
    p = len(values)
    if p == 1:
        return e.base(values[0])
    w = e.root(p.bit_length() - 1)
    xp1 = e.sub(e.pow(point, p), e.ONE)
    if not any(xp1):                                               # the point lies on the subgroup
        wi = 1
        for v in values:
            if point == e.base(wi):
                return e.base(v)
            wi = wi * w % e.P
        return e.ZERO
    acc, wi = e.ZERO, 1
    for v in values:
        acc = e.add(acc, e.scale(e.inverse(e.sub(point, e.base(wi))), v * wi % e.P))
        wi = wi * w % e.P
    return e.scale(e.mul(xp1, acc), e.inv(p))


def verify(config, air, proof, public_values=(), *, preprocessed_vk=None):
    """uni-stark verify.  `proof`: wire bytes, a uni_stark.Proof, or the dict proof_from_postcard returns.  `public_values`: canonical
    integers.  `air` supplies width(), num_public_values(), main_next_row_columns(), max_constraint_degree() and
    eval_folded_constraints(ext, local, next, public_values, is_first_row, is_last_row, is_transition, alpha) (the
    VerifierConstraintFolder, uni-stark/src/folder.rs); an AIR with preprocessed or periodic columns also supplies
    preprocessed_width(), preprocessed_next_row_columns(), periodic_columns() and takes the keywords preprocessed_local,
    preprocessed_next and periodic_values in its folder.  `preprocessed_vk`: uni_stark.PreprocessedVerifierKey, required iff the AIR
    has preprocessed columns.  `config.digest_codec` (default "f8") selects the wire form of digests: "u64x4" for the Keccak
    configuration (uni_stark.KeccakStarkConfig), "u8x32" for the SHA-256 configurations (uni_stark.Sha256StarkConfig).  Returns None; raises VerificationError."""
    from .uni_stark import get_log_num_quotient_chunks
    digest = getattr(config, "digest_codec", "f8")                # [F; 8] digests unless the configuration says otherwise
    if hasattr(proof, "to_postcard"):
        proof = proof.to_postcard()
    if isinstance(proof, (bytes, bytearray)):
        try:
            proof = proof_from_postcard(bytes(proof), config.pcs.dft.field.P, digest=digest)
        except ValueError as ex:
            raise VerificationError(f"malformed proof: {ex}") from None
    pcs = config.pcs
    params = pcs.fri
    e = Ext(pcs.dft.field)
    db = proof["degree_bits"]
    _need(db + params.log_blowup <= e.two_adicity, "degree bits out of range")
    n = 1 << db
    log_chunks = get_log_num_quotient_chunks(air)
    nchunks = 1 << log_chunks
    width = air.width()
    main_next = len(air.main_next_row_columns()) > 0
    _need(len(public_values) == air.num_public_values(), "public values length mismatch")
    _need(len(proof["trace_local"]) == width, "opened values dimension mismatch")
    if main_next:
        _need(proof["trace_next"] is not None and len(proof["trace_next"]) == width, "opened values dimension mismatch")
    else:
        _need(proof["trace_next"] is None, "opened values dimension mismatch")
    _need(len(proof["quotient_chunks"]) == nchunks and all(len(c) == 4 for c in proof["quotient_chunks"]), "opened values dimension mismatch")
    # process_preprocessed_trace (verifier.rs:203-277): the width is the key's, else the AIR's; the opened rows must match it
    pre_width = preprocessed_vk.width if preprocessed_vk is not None else int(getattr(air, "preprocessed_width", lambda: 0)())
    pre_next = len(getattr(air, "preprocessed_next_row_columns", lambda: [])()) > 0
    pre_local_v, pre_next_v = proof.get("preprocessed_local"), proof.get("preprocessed_next")
    _need((0 if pre_local_v is None else len(pre_local_v)) == pre_width
          and (0 if pre_next_v is None else len(pre_next_v)) == (pre_width if pre_next else 0), "preprocessed trace width mismatch")
    _need((pre_width == 0) == (preprocessed_vk is None), "preprocessed verifier key inconsistent with the AIR")
    if preprocessed_vk is not None:
        _need(preprocessed_vk.degree_bits == db, "preprocessed degree mismatch")
    periodic = [list(c) for c in getattr(air, "periodic_columns", lambda: [])()]
    from .air import periodic_column_error
    err = periodic_column_error(periodic, n)                       # check_periodic_column_lengths (verifier.rs:25-50)
    _need(err is None, f"invalid periodic column: {err}")

    ch = config.initialise_challenger()
    ch.observe_canonical(db); ch.observe_canonical(db); ch.observe_canonical(pre_width)     # degree_bits, base_degree_bits, preprocessed width
    _observe_cap(ch, proof["trace_commit"])
    if pre_width > 0:
        _observe_cap(ch, preprocessed_vk.commitment)
    for v in public_values:
        ch.observe_canonical(v)
    alpha = e.ec(ch.sample_algebra_element())
    _observe_cap(ch, proof["quotient_commit"])
    zeta = e.ec(ch.sample_algebra_element())
    z_h = e.sub(e.pow(zeta, n), e.ONE)
    _need(any(z_h), "out-of-domain point lies in the trace domain")
    g = e.root(db)
    zeta_next = e.scale(zeta, g)
    local = [e.ec(v) for v in proof["trace_local"]]
    nxt = [e.ec(v) for v in proof["trace_next"]] if main_next else [e.ZERO] * width
    chunks = [[e.ec(v) for v in c] for c in proof["quotient_chunks"]]
    trace_pts = [(zeta, local)] + ([(zeta_next, nxt)] if main_next else [])
    rounds = [(proof["trace_commit"], [(db, trace_pts)]), (proof["quotient_commit"], [(db, [(zeta, c)]) for c in chunks])]
    opened = [proof["trace_local"]] + ([proof["trace_next"]] if main_next else []) + list(proof["quotient_chunks"])
    pre_local, pre_nxt = None, None
    if pre_width > 0:                                              # the preprocessed round last
        pre_local = [e.ec(v) for v in pre_local_v]
        pre_nxt = [e.ec(v) for v in pre_next_v] if pre_next else [e.ZERO] * pre_width
        rounds.append((preprocessed_vk.commitment, [(db, [(zeta, pre_local)] + ([(zeta_next, pre_nxt)] if pre_next else []))]))
        opened += [pre_local_v] + ([pre_next_v] if pre_next else [])
    for ys in opened:                                              # TwoAdicFriPcs::verify: every opened value, in commitment order
        ch.observe_slice(np.asarray(ys, dtype=np.uint32))
    verify_fri(e, params, pcs.mmcs, proof, ch, rounds)

    # recompose_quotient_from_chunks: chunk i lives on GENERATOR * h^i * K, |K| = N, h of order N * chunks
    h = e.root(db + log_chunks)
    shifts = [e.GEN * pow(h, i, e.P) % e.P for i in range(nchunks)]
    van = lambda s, x: e.sub(e.pow(e.scale(x, e.inv(s)), n), e.ONE)
    quotient = [0, 0, 0, 0]
    for i in range(nchunks):
        zp = [1, 0, 0, 0]
        for j in range(nchunks):
            if j != i:
                zp = e.mul(zp, e.mul(van(shifts[j], zeta), e.inverse(van(shifts[j], e.base(shifts[i])))))
        quotient = e.add(quotient, e.mul(zp, e.from_basis(chunks[i])))
    ginv = e.inv(g)
    is_first = e.mul(z_h, e.inverse(e.sub(zeta, e.ONE)))                       # selectors_at_point, field/src/coset.rs
    is_last = e.mul(z_h, e.inverse(e.sub(zeta, e.base(ginv))))
    is_trans = e.sub(zeta, e.base(ginv))
    if pre_width > 0 or periodic:
        periodic_values = [eval_periodic_poly(e, col, e.pow(zeta, n // len(col))) for col in periodic]
        folded = air.eval_folded_constraints(e, local, nxt, list(public_values), is_first, is_last, is_trans, alpha,
                                             preprocessed_local=pre_local, preprocessed_next=pre_nxt, periodic_values=periodic_values)
    else:
        folded = air.eval_folded_constraints(e, local, nxt, list(public_values), is_first, is_last, is_trans, alpha)
    _need(e.mul(folded, e.inverse(z_h)) == quotient, "out-of-domain evaluation mismatch")
