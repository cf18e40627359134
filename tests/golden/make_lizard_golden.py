#!/usr/bin/env python3
"""Write tests/golden/lizard.json: the reference's Lizard known answers, copied as data, and point vectors computed by the
independent model (tests/lizard_model.py), each labelled with what it exercises.

The generator asserts that the model reproduces every reference known answer and that the C oracle
(tests/host/lizard_oracle.c) agrees with every vector.  Known answers (curve25519-dalek src/lizard/lizard_ristretto.rs):
  lizard_encode (:257-283, from testLizard() of vendor/ristretto.sage) and the elligator_inv corner inputs fe = 0 and
  fe = +sqrt(i d) (:309-317).

Point vectors ("points") carry the point as a CompressedRistretto ("ristretto") or as 20 radix-2^51 limbs of one
representative ("extended", used as given), and the expected lizard_decode (payload or null, status 0 Some / 1 None /
2 undecodable, n_found) and map_to_curve_inverse (16 candidates or null, and the mask)."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import h2c_model as H  # noqa: E402
import lizard_model as L  # noqa: E402

p = L.p

KATS = [  # (data, CompressedRistretto of lizard_encode::<Sha256>(data)), lizard_ristretto.rs:262-279
    ("00000000000000000000000000000000", "f0b7e34484f74cf00f15024b738539738646bbbe1e9bc7509a676815227e774f"),
    ("01010101010101010101010101010101", "cc92e81f585afc5caac88660d8d17e9025a44489a363042123f6af0702156e65"),
    ("000102030405060708090a0b0c0d0e0f", "c830573f8a8e7778671f76cdc796dc0a235cf177f197d9fcba06e84e96247444"),
    ("dddddddddddddddddddddddddddddddd", "ccb60554c081841037f821fa827b6a5bc2531f80e2647f1a858611f4ccfe3056"),
]
# fe = +sqrt(i d), the second corner input of elligator_inv (lizard_ristretto.rs:314-317)
SQRT_ID_BYTES = bytes([168, 27, 92, 74, 203, 42, 48, 117, 170, 109, 234, 14, 45, 169, 188, 205, 21, 110, 235, 115, 153, 84, 52,
                       117, 151, 235, 123, 244, 88, 85, 179, 5])


def point_record(label, P=None, enc=None):
    """A point vector: enc (CompressedRistretto bytes) or P (an extended representative, used as given)."""
    if enc is not None:
        Q = L.ristretto_decode(enc)
        rec = {"label": label, "fmt": "ristretto", "point": enc.hex()}
    else:
        Q = P
        rec = {"label": label, "fmt": "extended", "point": L.limbs_bytes(P).hex()}
    if Q is None:
        rec.update(decode=None, status=2, n_found=0, inverse=[None] * 16, mask=0)
        return rec
    data, n_found, _ = L.lizard_decode_detail(Q)
    inv = L.map_to_curve_inverse(Q)
    rec.update(decode=None if data is None else data.hex(), status=0 if data is not None else 1, n_found=n_found,
               inverse=[None if x is None else x.hex() for x in inv], mask=sum(1 << j for j, x in enumerate(inv) if x is not None))
    return rec


def jacobi_labels(P):
    """What the Jacobi points of P exercise: the X = 0 or Y = 0 case, s = 0 with t = 1 or t = -1."""
    out = []
    if L.x_or_y_is_zero(P):
        out.append("X = 0 or Y = 0")
    for k, (s, t) in enumerate(L.to_jacobi_quartic(P)):
        for lab, (ss, tt) in (("", (s, t)), ("dual ", ((-s) % p, (-t) % p))):
            if ss == 0:
                out.append("%sjc%d: s = 0, t = %s" % (lab, k, "1" if tt == 1 else ("-1" if tt == p - 1 else "?")))
    return out


def generate():
    rnd = random.Random(20261016)
    g = {}
    # ---- the reference's known answers, with where the encoded element sits (the representative map_to_curve returns)
    kats = []
    for data_hex, enc_hex in KATS:
        data = bytes.fromhex(data_hex)
        assert L.lizard_encode(data).hex() == enc_hex, data_hex
        assert L.lizard_decode(L.ristretto_decode(bytes.fromhex(enc_hex))) == data
        P = L.lizard_encode_point(data)
        _, n_found, slot = L.lizard_decode_detail(P)
        kats.append({"data": data_hex, "out": enc_hex, "slot": slot, "some": sum(x is not None for x in L.map_to_curve_inverse(P))})
    assert [k["slot"] for k in kats] == [1, 1, 1, 0] and [k["some"] for k in kats] == [6, 8, 12, 8]
    g["lizard_encode_kat"] = kats
    # ---- map_to_curve inputs: the elligator_inv corners (fe made even and below 2^255, as the reference's test does)
    maps = []
    for lab, b in (("fe = 0", bytes(32)), ("fe = +sqrt(i d)", SQRT_ID_BYTES)):
        b = bytearray(b); b[0] &= 254; b[31] &= 127; b = bytes(b)
        assert L.fe_from_bytes(b) == (0 if lab == "fe = 0" else L.SQRT_ID)
        maps.append({"label": lab, "in": b.hex(), "out": L.map_to_curve(b).hex()})
    for k in range(4):
        b = rnd.randbytes(32)
        maps.append({"label": "random, bit 255 %s" % ("set" if b[31] >> 7 else "clear"), "in": b.hex(), "out": L.map_to_curve(b).hex()})
    g["map_to_curve"] = maps
    # ---- e_inv_positive at the Jacobi level
    e_inv = []
    for lab, s, t in (("s = 0, t = 1", 0, 1), ("s = 0, t = -1", 0, p - 1)):
        e_inv.append((lab, s, t))
    sq_seen = {True: 0, False: 0}
    while min(sq_seen.values()) < 2:
        P = L.map_to_curve_point(rnd.randbytes(32))
        s, t = L.to_jacobi_quartic(P)[rnd.randrange(4)]
        x = L.e_inv_positive(s, t)
        if sq_seen[x is not None] < 2:
            sq_seen[x is not None] += 1
            e_inv.append(("a square root exists" if x is not None else "no square root", s, t))
    g["e_inv_positive"] = [{"label": lab, "s": L.fe_bytes(s).hex(), "t": L.fe_bytes(t).hex(),
                            "out": None if L.e_inv_positive(s, t) is None else L.fe_bytes(L.e_inv_positive(s, t)).hex()}
                           for lab, s, t in e_inv]
    # ---- point vectors
    pts = []
    for k in kats:
        data = bytes.fromhex(k["data"])
        pts.append(point_record("KAT %s: encoding" % k["data"], enc=bytes.fromhex(k["out"])))
        pts.append(point_record("KAT %s: map_to_curve representative, slot %d" % (k["data"], k["slot"]), P=L.lizard_encode_point(data)))
    for m in maps[:2]:
        P = L.map_to_curve_point(bytes.fromhex(m["in"]))
        for c, Q in enumerate(L.coset4(P)):
            rec = point_record("elligator_inv corner %s, coset representative %d (%s)" % (m["label"], c, "; ".join(jacobi_labels(Q))), P=Q)
            assert m["in"] in rec["inverse"], rec["label"]
            pts.append(rec)
    pts.append(point_record("identity encoding", enc=bytes(32)))
    for c, Q in enumerate(L.coset4(L.IDENTITY)):
        pts.append(point_record("identity, coset representative %d (%s)" % (c, "; ".join(jacobi_labels(Q))), P=Q))
    n_partial = n_none = 0
    while n_partial < 6 or n_none < 4:
        enc = H.from_uniform_bytes(rnd.randbytes(64))
        rec = point_record("random point; not a Lizard encoding", enc=enc)
        assert rec["status"] == 1                        # not a Lizard encoding
        if 0 < rec["mask"] < 0xffff and n_partial < 6:
            rec["label"] = "partial mask, %d of 16 Some; not a Lizard encoding" % bin(rec["mask"]).count("1")
            pts.append(rec); n_partial += 1
        elif rec["mask"] == 0 and n_none < 4:
            rec["label"] = "no candidate; not a Lizard encoding"
            pts.append(rec); n_none += 1
        elif n_none < 4 and rnd.random() < 0.02:
            pts.append(rec)
    # one Lizard point under several Z scalings: the pairs of candidates swap (the invsqrt picks the non-negative root)
    data = bytes(range(100, 116))
    P = L.ristretto_decode(L.lizard_encode(data))
    base = L.map_to_curve_inverse(P)
    reordered = 0
    lam_tried = 0
    while reordered < 3:
        lam = rnd.randrange(2, p)
        lam_tried += 1
        Q = L.scale(P, lam)
        rec = point_record("Lizard point scaled by lambda (%s)" % ("candidates reordered" if L.map_to_curve_inverse(Q) != base else "same order"), P=Q)
        assert rec["decode"] == data.hex()
        if L.map_to_curve_inverse(Q) != base:
            reordered += 1
            pts.append(rec)
        elif lam_tried < 4:
            pts.append(rec)
    pts.append(point_record("Lizard point, Z = 1 (the decoded representative)", P=P))
    for lab, enc in (("s = p (not canonical)", p.to_bytes(32, "little")), ("s = 1 (negative)", (1).to_bytes(32, "little")),
                     ("bit 255 set", bytes(31) + b"\x80"), ("all ones", b"\xff" * 32)):
        pts.append(point_record("undecodable: " + lab, enc=enc))
    n_sq = 0
    while n_sq < 2:
        s = rnd.randrange(0, p, 2)
        enc = s.to_bytes(32, "little")
        if L.ristretto_decode(enc) is None:
            pts.append(point_record("undecodable: even s, no square root", enc=enc)); n_sq += 1
    g["points"] = pts
    return g


def _pt(v):
    import lizard_oracle
    return bytes.fromhex(v["point"]), lizard_oracle.FMT_EXTENDED if v["fmt"] == "extended" else lizard_oracle.FMT_RISTRETTO


def check_oracle(g):
    import lizard_oracle
    o = lizard_oracle.load()
    for k in g["lizard_encode_kat"]:
        assert o.lizard_encode(bytes.fromhex(k["data"])).hex() == k["out"]
    for v in g["map_to_curve"]:
        assert o.map_to_curve_batch([bytes.fromhex(v["in"])])[0].hex() == v["out"], v["label"]
    for v in g["points"]:
        pt, fmt = _pt(v)
        st, data, n_found = o.lizard_decode(pt, fmt)
        assert st == v["status"] and n_found == v["n_found"], v["label"]
        assert data.hex() == (v["decode"] or "00" * 16), v["label"]
        bad, cands, mask = o.map_to_curve_inverse(pt, fmt)
        assert bad == (v["status"] == 2) and mask == v["mask"], v["label"]
        assert [c.hex() for c in cands] == [x or "00" * 32 for x in v["inverse"]], v["label"]


def render(g):
    return json.dumps(g, indent=1, sort_keys=True) + "\n"


if __name__ == "__main__":
    g = generate()
    check_oracle(g)
    path = os.path.join(HERE, "lizard.json")
    with open(path, "w") as f:
        f.write(render(g))
    print("wrote", path, {k: len(v) for k, v in g.items() if isinstance(v, list)})
