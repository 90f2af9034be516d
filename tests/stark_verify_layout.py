"""CPU restatement of the reference verifier for AIRs with preprocessed and periodic columns — test infrastructure.

`verify` is tests/stark_verify.py's `verify` (uni-stark/src/verifier.rs:282-561) extended as verify_with_preprocessed does:

    process_preprocessed_trace (:203-277)   the width is the verifier key's, else the AIR's; the opened preprocessed rows must have it
                                            (and the next row only when preprocessed_next_row_columns is not empty); a key is given
                                            iff the width is not 0, with the trace's degree bits
    check_periodic_column_lengths (:25-50)  every period a power of two, at most the trace length
    transcript (:405-425)                   degree bits, preprocessed width, trace cap, preprocessed cap (width > 0), public values
    rounds (:508-520)                       the preprocessed round last, at zeta (and zeta * omega)
    periodic values at zeta                 P_j(zeta^(n / p_j)) in plain Lagrange form over the subgroup of size p_j (not the
                                            barycentric form the product verifier uses)

Everything else (FRI, MMCS, challenger, field arithmetic) is stark_verify's, itself pinned on the reference's committed proof."""
from stark_verify import Challenger, VerifyError, _need, verify_fri  # noqa: F401  (VerifyError re-exported for callers)


def periodic_at(f, values, point):
    """The degree < p interpolant of `values` over the subgroup of size p, at an EF point: plain Lagrange form."""
    p = len(values)
    w = f.root(p.bit_length() - 1)
    xs = [pow(w, i, f.P) for i in range(p)]
    acc = [0, 0, 0, 0]
    for i, v in enumerate(values):
        num, den = [1, 0, 0, 0], 1
        for j in range(p):
            if j != i:
                num = f.emul(num, f.esub(point, f.ebase(xs[j])))
                den = den * (xs[i] - xs[j]) % f.P
        acc = f.eadd(acc, f.escal(num, v * f.inv(den) % f.P))
    return acc


def verify(f, cfg, air, proof, public_values=(), preprocessed_vk=None):
    """uni-stark verify_with_preprocessed.  `cfg` as stark_verify.verify.  `air`: dict(width, main_next, log_quotient_chunks,
    num_public_values, preprocessed_width, preprocessed_next (bool), periodic (columns of canonical values), constraints(f, local, nxt,
    public_values, is_first, is_last, is_transition, alpha, preprocessed_local, preprocessed_next, periodic_values) -> folded EF).
    `preprocessed_vk`: dict(width, degree_bits, commitment) or None.  `proof`: proof_from_postcard(...).  Raises VerifyError."""
    db = proof["degree_bits"]
    _need(0 <= db and db + cfg["log_blowup"] <= f.two_adicity, "degree bits out of range")
    n = 1 << db
    nchunks = 1 << air["log_quotient_chunks"]
    _need(len(public_values) == air["num_public_values"], "public values length")
    _need(len(proof["trace_local"]) == air["width"], "trace_local width")
    if air["main_next"]:
        _need(proof["trace_next"] is not None and len(proof["trace_next"]) == air["width"], "trace_next width")
    else:
        _need(proof["trace_next"] is None, "unexpected trace_next")
    _need(len(proof["quotient_chunks"]) == nchunks and all(len(c) == 4 for c in proof["quotient_chunks"]), "quotient chunk shape")
    pw = preprocessed_vk["width"] if preprocessed_vk is not None else air.get("preprocessed_width", 0)
    pnext = air.get("preprocessed_next", False)
    pl, pn = proof.get("preprocessed_local"), proof.get("preprocessed_next")
    _need((0 if pl is None else len(pl)) == pw and (0 if pn is None else len(pn)) == (pw if pnext else 0), "preprocessed width")
    _need((pw == 0) == (preprocessed_vk is None), "preprocessed key")
    _need(preprocessed_vk is None or preprocessed_vk["degree_bits"] == db, "preprocessed degree")
    periodic = air.get("periodic", [])
    for col in periodic:
        _need(len(col) > 0 and len(col) & (len(col) - 1) == 0 and len(col) <= n, "periodic column length")
    ch = Challenger(f, cfg["challenger_perm"], cfg["challenger_width"], cfg["challenger_rate"])
    ch.observe(db); ch.observe(db); ch.observe(pw)
    ch.observe_words(proof["trace_commit"])
    if pw:
        ch.observe_words(preprocessed_vk["commitment"])
    for v in public_values:
        ch.observe(v)
    alpha = ch.sample_ef()
    ch.observe_words(proof["quotient_commit"])
    zeta = ch.sample_ef()
    z_h = f.esub(f.epow(zeta, n), [1, 0, 0, 0])
    _need(any(z_h), "out-of-domain point lies in the trace domain")
    g = f.root(db)
    zeta_next = f.escal(zeta, g)
    can = lambda rows: [[f.c(v) for v in e] for e in rows]
    local, nxt = can(proof["trace_local"]), (can(proof["trace_next"]) if air["main_next"] else [[0, 0, 0, 0]] * air["width"])
    chunks = [can(c) for c in proof["quotient_chunks"]]
    trace_pts = [(zeta, local)] + ([(zeta_next, nxt)] if air["main_next"] else [])
    rounds = [(proof["trace_commit"], [(db, trace_pts)]), (proof["quotient_commit"], [(db, [(zeta, c)]) for c in chunks])]
    pre_local = pre_nxt = None
    if pw:
        pre_local = can(pl)
        pre_nxt = can(pn) if pnext else [[0, 0, 0, 0]] * pw
        rounds.append((preprocessed_vk["commitment"], [(db, [(zeta, pre_local)] + ([(zeta_next, pre_nxt)] if pnext else []))]))
    for _, mats in rounds:                                       # TwoAdicFriPcs::verify: all opened values enter the transcript first
        for _, pts in mats:
            for _, ys in pts:
                for e in ys:
                    for v in e:
                        ch.observe(v)
    verify_fri(f, cfg, proof, ch, rounds)
    h = f.root(db + air["log_quotient_chunks"])
    shifts = [f.GEN * pow(h, i, f.P) % f.P for i in range(nchunks)]
    van = lambda s, x: f.esub(f.epow(f.escal(x, f.inv(s)), n), [1, 0, 0, 0])
    quotient = [0, 0, 0, 0]
    for i in range(nchunks):
        zp = [1, 0, 0, 0]
        for j in range(nchunks):
            if j != i:
                zp = f.emul(zp, f.emul(van(shifts[j], zeta), f.einv(van(shifts[j], f.ebase(shifts[i])))))
        quotient = f.eadd(quotient, f.emul(zp, f.from_basis(chunks[i])))
    ginv = f.inv(g)
    is_first = f.emul(z_h, f.einv(f.esub(zeta, [1, 0, 0, 0])))
    is_last = f.emul(z_h, f.einv(f.esub(zeta, f.ebase(ginv))))
    is_trans = f.esub(zeta, f.ebase(ginv))
    per = [periodic_at(f, col, f.epow(zeta, n // len(col))) for col in periodic]
    folded = air["constraints"](f, local, nxt, list(public_values), is_first, is_last, is_trans, alpha, pre_local, pre_nxt, per)
    _need(f.emul(folded, f.einv(z_h)) == quotient, "out-of-domain evaluation mismatch")
