#!/usr/bin/env python3
"""Write tests/golden/scalar_ops.json: the known answers of curve25519-dalek's Scalar tests (src/scalar.rs), read out of
the reference's source as data, each checked here with Python integers so that the fixture checks itself where the
reference is absent (check()).

    python3 tests/golden/make_scalar_golden.py <curve25519-dalek checkout>

Read from scalar.rs: the from_hash doc example (its message and digest scalar), the statics X, XINV, Y and X_TIMES_Y,
the expected values of impl_sum and impl_product, the three encodings of canonical_decoding; div_by_2, invert and
neg_twice_is_identity give their cases as the tests run them."""
import hashlib
import json
import os
import re
import sys

L = 2**252 + 27742317777372353535851937790883648493
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "scalar_ops.json")


def _line(src, pos):
    return "curve25519-dalek/src/scalar.rs:%d" % (src.count("\n", 0, pos) + 1)


def _bytes_array(text):
    vals = [int(v, 0) for v in re.findall(r"0x[0-9a-fA-F]+|\d+", text)]
    assert len(vals) == 32, vals
    return bytes(vals)


def _static(src, name):
    m = re.search(r"static %s: Scalar = Scalar \{\s*bytes: \[(.*?)\]," % name, src, re.S)
    return _bytes_array(m.group(1)).hex(), _line(src, m.start())


def _fn_body(src, name):
    m = re.search(r"fn %s\(\) \{(.*?)\n    \}\n" % name, src, re.S)
    return m.group(1), _line(src, m.start())


def le(x):
    return x.to_bytes(32, "little").hex()


def make(src):
    out = {}
    for name in ("X", "XINV", "Y", "X_TIMES_Y"):
        out[name] = dict(zip(("hex", "src"), _static(src, name)))
    # from_hash doc example: the chained strings are the message
    m = re.search(r"let mut h = Sha512::new\(\)(.*?)let s = Scalar::from_hash\(h\);.*?s\.to_bytes\(\),\s*///\s*\[(.*?)\],", src, re.S)
    msg = "".join(re.findall(r'\.chain\("(.*?)"\)', m.group(1))).encode()
    digest = _bytes_array(re.sub(r"///", "", m.group(2)))
    out["from_hash"] = {"message": msg.hex(), "scalar": digest.hex(), "src": _line(src, m.start())}
    # impl_sum / impl_product: the u64 values they compare against, with the inputs the tests fold
    body, where = _fn_body(src, "impl_sum")
    want = [int(v) for v in re.findall(r"Scalar::from\((\d+)u64\)", body)]
    assert want == [2, 1, 2, 10, 20, 30], want
    out["impl_sum"] = {"src": where, "cases": [
        {"items": [le(1), le(1)], "sum": le(2)}, {"items": [], "sum": le(0)},
        {"items": [le(1)] * 10, "sum": le(10)}, {"items": [le(2)] * 10, "sum": le(20)}, {"items": [le(3)] * 10, "sum": le(30)}]}
    body, where = _fn_body(src, "impl_product")
    want = [int(v) for v in re.findall(r"Scalar::from\((\d+)u64\)", body)]
    assert want == [2, 3, 1024, 59049, 60466176], want
    x, y = out["X"]["hex"], out["Y"]["hex"]
    out["impl_product"] = {"src": where, "cases": [
        {"items": [x, y], "product": out["X_TIMES_Y"]["hex"]}, {"items": [], "product": le(1)},
        {"items": [le(2)] * 10, "product": le(1024)}, {"items": [le(3)] * 10, "product": le(59049)},
        {"items": [le(6)] * 10, "product": le(60466176)}]}
    # div_by_2: 0..31 and -0..-31, each d with d + d = s
    _, where = _fn_body(src, "div_by_2")
    inv2 = (L + 1) // 2
    cases = [i for i in range(32)] + [(-i) % L for i in range(32)]
    out["div_by_2"] = {"src": where, "cases": [{"s": le(s), "half": le(s * inv2 % L)} for s in cases]}
    _, where = _fn_body(src, "invert")
    out["invert"] = {"src": where, "s": x, "inv": out["XINV"]["hex"]}
    _, where = _fn_body(src, "neg_twice_is_identity")
    out["neg_twice_is_identity"] = {"src": where, "s": x, "neg": le((-int.from_bytes(bytes.fromhex(x), "little")) % L)}
    # canonical_decoding: one canonical encoding, one unreduced, one with the high bit set
    body, where = _fn_body(src, "canonical_decoding")
    arrays = re.findall(r"let (\w+) = \[(.*?)\];", body, re.S)
    enc = {}
    for name, text in arrays:
        if ";" in text:                                    # [16; 32]
            v, k = text.split(";")
            enc[name] = bytes([int(v)] * int(k))
        else:
            enc[name] = _bytes_array(text)
    out["canonical_decoding"] = {"src": where, "cases": [
        {"bytes": enc["canonical_bytes"].hex(), "canonical": True},
        {"bytes": enc["non_canonical_bytes_because_unreduced"].hex(), "canonical": False},
        {"bytes": enc["non_canonical_bytes_because_highbit"].hex(), "canonical": False}]}
    check(out)
    return out


def check(g):
    """Every value of the fixture against Python integers mod l."""
    n = lambda h: int.from_bytes(bytes.fromhex(h), "little")   # noqa: E731
    X, Y = n(g["X"]["hex"]), n(g["Y"]["hex"])
    assert X * n(g["XINV"]["hex"]) % L == 1 and X * Y % L == n(g["X_TIMES_Y"]["hex"])
    digest = hashlib.sha512(bytes.fromhex(g["from_hash"]["message"])).digest()
    assert int.from_bytes(digest, "little") % L == n(g["from_hash"]["scalar"])
    for c in g["impl_sum"]["cases"]:
        assert sum(n(v) for v in c["items"]) % L == n(c["sum"])
    for c in g["impl_product"]["cases"]:
        p = 1
        for v in c["items"]:
            p = p * n(v) % L
        assert p == n(c["product"])
    for c in g["div_by_2"]["cases"]:
        assert 2 * n(c["half"]) % L == n(c["s"]) and n(c["half"]) < L
    assert n(g["invert"]["s"]) * n(g["invert"]["inv"]) % L == 1
    assert (n(g["neg_twice_is_identity"]["s"]) + n(g["neg_twice_is_identity"]["neg"])) % L == 0
    for c in g["canonical_decoding"]["cases"]:
        assert (n(c["bytes"]) < L) == c["canonical"]


if __name__ == "__main__":
    with open(os.path.join(sys.argv[1], "src", "scalar.rs")) as f:
        fixture = make(f.read())
    with open(OUT, "w") as f:
        json.dump(fixture, f, indent=1)
        f.write("\n")
