"""Writes tests/golden/ristretto.json: CompressedRistretto encodings labelled with the rejection terms they fire.

CompressedRistretto::decompress (curve25519-dalek ristretto.rs:266-345) returns None when any of five terms holds:

  noncanonical   the bytes are not the encoding of their own field element (s >= p, or bit 255 set; the field
                 element is read like FieldElement::from_bytes, which ignores bit 255)
  negative       s is negative (odd)
  nonsquare      invsqrt(v u2^2) finds no square root
  t_negative     t = x y is negative
  y_zero         y = 0

`decode_terms` restates the decode in plain big integers and returns the set of terms that fire.  A decoder that
drops one term is only seen through a vector where that term fires alone, so every class holds at least 16 such
single-term vectors, or every candidate there is:

  noncanonical   all 19 values s in [p, 2^255), and the 16 small multiples with bit 255 set
  negative       p - s for 16 valid even s (decodes like s but for the sign of s), and the bytes of EDWARDS_D
                 (ristretto.rs decompress_negative_s_fails)
  nonsquare,     even canonical s drawn at random, sorted by their term sets (the survey of 1024 draws is recorded)
  t_negative
  y_zero         s = p - 1, the only s with y = 0 that fires nothing else (y = 0 needs s^2 = 1, where s = 1 is
                 negative, or invsqrt(0), which also fires nonsquare); and the even s where invsqrt(0) happens
  valid          the 16 small multiples of kat.json and 16 encodings of random multiples of the basepoint

Every label comes from `decode_terms`, and the C oracle must reject exactly the vectors with a term."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

P = 2**255 - 19
D = (-121665 * pow(121666, P - 2, P)) % P
SQRT_M1 = pow(2, (P - 1) // 4, P)
TERMS = ["noncanonical", "negative", "nonsquare", "t_negative", "y_zero"]
SINGLES = 16                       # single-term vectors wanted per class
SURVEY = 1024                      # random even canonical s drawn for the nonsquare / t_negative classes


def sqrt_ratio_i(u, v):
    """FieldElement::sqrt_ratio_i (field.rs): (u/v is a non-zero square, the non-negative root of u/v or i u/v)"""
    v3 = v * v * v % P
    v7 = v3 * v3 * v % P
    r = u * v3 * pow(u * v7 % P, (P - 5) // 8, P) % P
    check = v * r * r % P
    correct, flipped, flipped_i = check == u % P, check == -u % P, check == -u * SQRT_M1 % P
    if flipped or flipped_i:
        r = r * SQRT_M1 % P
    if r & 1:
        r = P - r
    return correct or flipped, r


def decode_terms(enc):
    """the terms of CompressedRistretto::decompress that fire for the 32 bytes `enc`, in TERMS order"""
    s = (int.from_bytes(enc, "little") & (2**255 - 1)) % P
    fired = set()
    if s.to_bytes(32, "little") != enc:
        fired.add("noncanonical")
    if s & 1:
        fired.add("negative")
    ss = s * s % P
    u1, u2 = (1 - ss) % P, (1 + ss) % P
    u2_sqr = u2 * u2 % P
    v = (-D * u1 * u1 - u2_sqr) % P
    ok, inv = sqrt_ratio_i(1, v * u2_sqr % P)
    dx = inv * u2 % P
    dy = inv * dx * v % P
    x = 2 * s * dx % P
    if x & 1:
        x = P - x
    y = u1 * dy % P
    if not ok:
        fired.add("nonsquare")
    if x * y % P & 1:
        fired.add("t_negative")
    if y == 0:
        fired.add("y_zero")
    return [t for t in TERMS if t in fired]


def sqrt_mod_p(a):
    """the roots of a mod p (p = 5 mod 8), [] if a is not a square"""
    a %= P
    r = pow(a, (P + 3) // 8, P)
    if r * r % P != a:
        r = r * SQRT_M1 % P
    return sorted({r, (P - r) % P}) if r * r % P == a else []


def b32(x):
    return x.to_bytes(32, "little")


def build_doc():
    import oracle_lib
    orc = oracle_lib.load()
    with open(os.path.join(HERE, "kat.json")) as f:
        kat = json.load(f)
    rnd = random.Random(0x5255)
    small = [bytes.fromhex(h) for h in kat["ristretto"]["SMALL_MULTIPLES"]["hex"]]
    B = orc.basepoint()
    rand_valid = [orc.ristretto_compress(orc.scalarmul(b32(rnd.randrange(1, 2**252)), B)) for _ in range(SINGLES)]
    valid_even = [e for e in small[1:] + rand_valid]                    # every canonical encoding is even

    d_limbs = kat["u64_constants"]["EDWARDS_D"]["limbs"]
    edwards_d = b32(sum(l << (51 * i) for i, l in enumerate(d_limbs)))
    assert int.from_bytes(edwards_d, "little") == D

    survey = {}
    drawn = []
    for _ in range(SURVEY):
        s = rnd.randrange(P) & ~1
        terms = decode_terms(b32(s))
        survey["+".join(terms) or "valid"] = survey.get("+".join(terms) or "valid", 0) + 1
        drawn.append((b32(s), terms))

    def first(cands, term, k=SINGLES):
        return [e for e, t in cands if t == [term]][:k]

    ns_mixed = [e for e, t in drawn if "nonsquare" in t and t != ["nonsquare"]][:4]
    i_roots = [r for r in sqrt_mod_p(-1) if r % 2 == 0]                  # u2 = 0
    v_roots = [r for c in sqrt_mod_p(-D) for r in sqrt_mod_p((c - 1) * pow(c + 1, P - 2, P)) if r % 2 == 0]   # v = 0
    classes = {
        "noncanonical": [b32(s) for s in range(P, 2**255)] + [e[:31] + bytes([e[31] | 0x80]) for e in small],
        "negative": [b32(P - int.from_bytes(e, "little")) for e in valid_even[:SINGLES]] + [edwards_d],
        "nonsquare": first(drawn, "nonsquare") + ns_mixed,
        "t_negative": first(drawn, "t_negative"),
        "y_zero": [b32(P - 1)] + [b32(r) for r in i_roots + v_roots],
        "valid": small + rand_valid,
    }
    out = {}
    for name, encs in classes.items():
        out[name] = []
        for e in encs:
            terms = decode_terms(e)
            assert (orc.ristretto_decompress(e) is None) == bool(terms), (name, e.hex(), terms)
            assert (name == "valid") == (not terms) and (name == "valid" or name in terms), (name, e.hex(), terms)
            out[name].append({"s": e.hex(), "terms": terms})
    for term in TERMS:
        singles = sum(v["terms"] == [term] for v in out[term])
        assert singles >= SINGLES or term == "y_zero", (term, singles)
    return {"terms": TERMS, "even_s_survey": {"drawn": SURVEY, "by_terms": dict(sorted(survey.items()))},
            "classes": out}


def render(doc):
    return json.dumps(doc, indent=1) + "\n"


def main():
    with open(os.path.join(HERE, "ristretto.json"), "w") as f:
        f.write(render(build_doc()))


if __name__ == "__main__":
    main()
