"""Writes tests/golden/scalar_mul.json: variable-base scalar multiplication vectors of curve25519-dalek.

Transcribed from the reference's tests and constants:
  * A_SCALAR, B_SCALAR and A_TIMES_BASEPOINT (curve25519-dalek/src/edwards.rs, mod test);
  * BASEPOINT_ORDER, whose multiple of the basepoint is the identity (basepoint_mult_by_basepoint_order);
  * EIGHT_TORSION (src/backend/serial/u64/constants.rs) as radix-2^51 limbs.
Computed here with the C oracle (oracle/curve.c): A_SCALAR * A_TIMES_BASEPOINT, and the CompressedEdwardsY encodings of
the torsion points.  Run from the repository root: python tests/golden/make_scalar_mul_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))

A_SCALAR = "1a0e978a90f6622d3747023f8ad8264da758aa1b88e040d1589e7b7f2376ef09"
B_SCALAR = "91267acf25c2091ba217747b66f0b32e9df2a56741cfdac456a7d4aab8608a05"
A_TIMES_BASEPOINT = "ea27e26053df1b5956f14d5dec3c34c384a269b74cc3803ea8e2e7c9425e40a5"
BASEPOINT_ORDER = "edd3f55c1a631258d69cf7a2def9de1400000000000000000000000000000010"
BASEPOINT = "5866666666666666666666666666666666666666666666666666666666666666"
EIGHT_TORSION = [
    {"X": [0, 0, 0, 0, 0], "Y": [1, 0, 0, 0, 0], "Z": [1, 0, 0, 0, 0], "T": [0, 0, 0, 0, 0]},
    {"X": [358744748052810, 1691584618240980, 977650209285361, 1429865912637724, 560044844278676], "Y": [84926274344903, 473620666599931, 365590438845504, 1028470286882429, 2146499180330972], "Z": [1, 0, 0, 0, 0], "T": [1448326834587521, 1857896831960481, 1093722731865333, 1677408490711241, 1915505153018406]},
    {"X": [533094393274173, 2016890930128738, 18285341111199, 134597186663265, 1486323764102114], "Y": [0, 0, 0, 0, 0], "Z": [1, 0, 0, 0, 0], "T": [0, 0, 0, 0, 0]},
    {"X": [358744748052810, 1691584618240980, 977650209285361, 1429865912637724, 560044844278676], "Y": [2166873539340326, 1778179147085316, 1886209374839743, 1223329526802818, 105300633354275], "Z": [1, 0, 0, 0, 0], "T": [803472979097708, 393902981724766, 1158077081819914, 574391322974006, 336294660666841]},
    {"X": [0, 0, 0, 0, 0], "Y": [2251799813685228, 2251799813685247, 2251799813685247, 2251799813685247, 2251799813685247], "Z": [1, 0, 0, 0, 0], "T": [0, 0, 0, 0, 0]},
    {"X": [1893055065632419, 560215195444267, 1274149604399886, 821933901047523, 1691754969406571], "Y": [2166873539340326, 1778179147085316, 1886209374839743, 1223329526802818, 105300633354275], "Z": [1, 0, 0, 0, 0], "T": [1448326834587521, 1857896831960481, 1093722731865333, 1677408490711241, 1915505153018406]},
    {"X": [1718705420411056, 234908883556509, 2233514472574048, 2117202627021982, 765476049583133], "Y": [0, 0, 0, 0, 0], "Z": [1, 0, 0, 0, 0], "T": [0, 0, 0, 0, 0]},
    {"X": [1893055065632419, 560215195444267, 1274149604399886, 821933901047523, 1691754969406571], "Y": [84926274344903, 473620666599931, 365590438845504, 1028470286882429, 2146499180330972], "Z": [1, 0, 0, 0, 0], "T": [803472979097708, 393902981724766, 1158077081819914, 574391322974006, 336294660666841]},
]


def main():
    import oracle_lib
    orc = oracle_lib.load()
    a = bytes.fromhex(A_SCALAR)
    P = orc.decompress(bytes.fromhex(A_TIMES_BASEPOINT))
    assert orc.compress(orc.scalarmul(a, orc.basepoint())).hex() == A_TIMES_BASEPOINT
    assert orc.is_identity(orc.scalarmul(bytes.fromhex(BASEPOINT_ORDER), orc.basepoint()))
    torsion = []
    for t in EIGHT_TORSION:
        limbs = t["X"] + t["Y"] + t["Z"] + t["T"]
        torsion.append({"limbs": limbs, "compressed": orc.compress(orc.p3_from_limbs(limbs)).hex()})
    out = {
        "A_SCALAR": A_SCALAR,
        "B_SCALAR": B_SCALAR,
        "BASEPOINT": BASEPOINT,
        "A_TIMES_BASEPOINT": A_TIMES_BASEPOINT,
        "A_TIMES_A_TIMES_BASEPOINT": orc.compress(orc.scalarmul(a, P)),
        "BASEPOINT_ORDER": BASEPOINT_ORDER,
        "IDENTITY": "01" + "00" * 31,
        "EIGHT_TORSION": torsion,
    }
    out["A_TIMES_A_TIMES_BASEPOINT"] = out["A_TIMES_A_TIMES_BASEPOINT"].hex()
    with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
