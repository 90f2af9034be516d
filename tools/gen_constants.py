#!/usr/bin/env python3
"""Extract numeric parameters and known-answer vectors from the reference tree.

Run once as `python tools/gen_constants.py <Plonky3 checkout>`; outputs are committed:
  plonky3_b200/p2_constants.json   Poseidon2 round constants (canonical form) for
                                   BabyBear/KoalaBear widths 16 and 24
                                   (baby-bear/src/poseidon2.rs:111-281, koala-bear/src/poseidon2.rs:119-285)
  tests/golden/poseidon2_kat.json  known-answer vectors of the default-constant permutations
                                   (koala-bear/src/poseidon2.rs:614-653, baby-bear/src/poseidon2.rs:599-639)
  tests/golden/two_adic_generators.json  (baby_bear.rs:48-53, koala_bear.rs:73-78)
  tests/golden/poseidon1_constants.json  width-16 Poseidon1 of both fields (baby-bear/src/poseidon1.rs, koala-bear/src/poseidon1.rs,
                                   {baby-bear,koala-bear}/src/mds.rs): rounds, S-box degree, the circulant MDS's first column,
                                   the raw round constants and the known answer for input 0..15
Only numbers are extracted, no code.
"""
import json, re, sys, pathlib

REF = pathlib.Path(sys.argv[1])
OUT = pathlib.Path(__file__).resolve().parent.parent


def ints(s):
    return [int(x, 0) for x in re.findall(r"0x[0-9a-fA-F]+|\b\d+\b", s)]


def const_block(src, name):
    i = src.index("pub const " + name)
    j = src.index(";\n", src.index("=", i))
    body = src[src.index("=", i) + 1 : j]
    body = body[body.index("(") :]          # drop `KoalaBear::new_2d_array`
    return ints(body)


def kat(src, fn):
    i = src.index("fn " + fn)
    blk = src[i : src.index("assert_eq!", i)]
    a = blk.index("new_array(")
    b = blk.index("new_array(", a + 1)
    inp = ints(blk[a : blk.index("]);", a)][0:])
    exp = ints(blk[b : blk.index("]);", b)][0:])
    return inp, exp


def main():
    consts, kats, gens = {}, {}, {}
    for fld, d, pfx in (("baby_bear", "baby-bear", "BABYBEAR"), ("koala_bear", "koala-bear", "KOALABEAR")):
        src = (REF / d / "src" / "poseidon2.rs").read_text()
        for w in (16, 24):
            ini = const_block(src, f"{pfx}_POSEIDON2_RC_{w}_EXTERNAL_INITIAL")
            fin = const_block(src, f"{pfx}_POSEIDON2_RC_{w}_EXTERNAL_FINAL")
            itl = const_block(src, f"{pfx}_POSEIDON2_RC_{w}_INTERNAL")
            # first two ints of each block come from the type annotation "[[F; w]; 4]" / "[F; n]"
            ini = ini[-4 * w :]; fin = fin[-4 * w :]
            rp = int(re.search(rf"{pfx}_POSEIDON2_PARTIAL_ROUNDS_{w}: usize = (\d+)", src).group(1))
            itl = itl[-rp:]
            assert len(ini) == 4 * w and len(fin) == 4 * w and len(itl) == rp
            consts[f"{fld}_{w}"] = {"external_initial": ini, "external_final": fin, "internal": itl}
            name = "babybear" if fld == "baby_bear" else "koalabear"
            inp, exp = kat(src, f"test_default_{name}_poseidon2_width_{w}")
            assert len(inp) == w and len(exp) == w, (len(inp), len(exp))
            kats[f"{fld}_{w}"] = {"input": inp, "expected": exp}
        fsrc = (REF / d / "src" / f"{fld}.rs").read_text()
        i = fsrc.index("const TWO_ADIC_GENERATORS")
        blk = fsrc[i : fsrc.index("]);", i)]
        gens[fld] = ints(blk[blk.index("new_array(") :])
    (OUT / "plonky3_b200" / "p2_constants.json").write_text(json.dumps(consts))
    (OUT / "tests" / "golden" / "poseidon2_kat.json").write_text(json.dumps(kats, indent=0))
    (OUT / "tests" / "golden" / "two_adic_generators.json").write_text(json.dumps(gens))
    p1 = poseidon1()
    (OUT / "tests" / "golden" / "poseidon1_constants.json").write_text(json.dumps(p1, indent=0))
    print({k: (len(v["external_initial"]), len(v["internal"])) for k, v in consts.items()}, {k: len(v) for k, v in gens.items()},
          {k: (v["rounds_f"], v["rounds_p"], v["sbox_degree"]) for k, v in p1.items() if k != "note"})


def poseidon1():
    """The width-16 Poseidon1 instances of prove_prime_field_31 -o poseidon-1-permutations (examples/examples/prove_prime_field_31.rs)."""
    out = {"note": "width-16 Poseidon1; canonical values; mds_circ_col is the circulant MDS's first COLUMN, "
                   "first_row_to_first_col of the first row in mds.rs (col[0] = row[0], col[i] = row[16 - i]); "
                   "round_constants: rounds_f / 2 initial full rounds, rounds_p partial rounds, rounds_f / 2 terminal full rounds"}
    for fld, d, pfx, half, part in (("baby_bear", "baby-bear", "BABYBEAR", "BABYBEAR_POSEIDON1_HALF_FULL_ROUNDS", "BABYBEAR_POSEIDON1_PARTIAL_ROUNDS_16"),
                                    ("koala_bear", "koala-bear", "KOALABEAR", "KOALABEAR_POSEIDON_HALF_FULL_ROUNDS",
                                     "KOALABEAR_POSEIDON_PARTIAL_ROUNDS_16")):
        src = (REF / d / "src" / "poseidon1.rs").read_text()
        num = lambda name: int(re.search(rf"pub const {name}: \w+ = (\d+);", src).group(1))
        rounds_f, rounds_p, degree = 2 * num(half), num(part), num(f"{pfx}_S_BOX_DEGREE")
        i = src.index(f"pub const {pfx}_POSEIDON1_RC_16")
        blk = src[i: src.index("]);", i)]
        rc = ints(re.sub(r"//[^\n]*", "", blk[blk.index("new_2d_array(") + len("new_2d_array("):]))
        assert len(rc) == 16 * (rounds_f + rounds_p), len(rc)
        mds = (REF / d / "src" / "mds.rs").read_text()
        j = mds.index("MATRIX_CIRC_MDS_16_COL")
        row = ints(mds[mds.index("&[", j) + 1: mds.index("])", j)])
        assert len(row) == 16
        col = [row[0]] + [row[16 - k] for k in range(1, 16)]
        t = src.index("fn test_poseidon_width_16")
        tb = src[t: src.index("assert_eq!", t)]
        a = tb.index("new_array(")
        b = tb.index("new_array(", a + 1)
        kin, kout = ints(tb[a + 10: tb.index("]);", a)]), ints(tb[b + 10: tb.index("]);", b)])
        assert kin == list(range(16)) and len(kout) == 16
        out[fld] = {"width": 16, "rounds_f": rounds_f, "rounds_p": rounds_p, "sbox_degree": degree, "mds_circ_col": col,
                    "round_constants": [rc[16 * r: 16 * r + 16] for r in range(rounds_f + rounds_p)],
                    "kat_input": kin, "kat_expected": kout}
    return out


if __name__ == "__main__":
    main()
