"""CPU checks of the Lizard fixtures: the golden file is what its generator writes, the model reproduces the reference's
known answers, the model's and the C oracle's constants are their definitions, and the C oracle equals the model on
every vector and on random items (encode, decode and the inverse, CompressedRistretto and extended input with random Z)."""
import hashlib
import json
import os
import random
import sys

import pytest

import h2c_model as H
import lizard_oracle
import lizard_model as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_lizard_golden as G  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "lizard.json")) as f:
        return f.read()


@pytest.fixture(scope="module")
def ho():
    return lizard_oracle.load()


def test_file_is_what_the_generator_writes(golden):
    assert G.render(G.generate()) == golden


def test_model_reproduces_reference_kats():
    for data, enc in G.KATS:
        assert L.lizard_encode(bytes.fromhex(data)).hex() == enc
        P = L.ristretto_decode(bytes.fromhex(enc))
        assert L.lizard_decode(P) == bytes.fromhex(data)
        for Q in L.coset4(P):                        # every representative decodes the same
            assert L.lizard_decode(Q) == bytes.fromhex(data)
    # where the encoded element sits for the representative map_to_curve returns, and how many candidates are Some
    slots = [L.lizard_decode_detail(L.lizard_encode_point(bytes.fromhex(d)))[2] for d, _ in G.KATS]
    some = [sum(x is not None for x in L.map_to_curve_inverse(L.lizard_encode_point(bytes.fromhex(d)))) for d, _ in G.KATS]
    assert slots == [1, 1, 1, 0] and some == [6, 8, 12, 8]
    # the identity: all 16 candidates Some, with repeats, and no payload
    inv = L.map_to_curve_inverse(L.IDENTITY)
    assert all(x is not None for x in inv) and len(set(inv)) < 16
    assert L.lizard_decode(L.IDENTITY) is None


def test_elligator_inverse_corners_and_round_trip():
    """elligator_inv (lizard_ristretto.rs:303-344): the input is among the candidates of each coset representative, and
    every candidate maps back to the point."""
    rnd = random.Random(5)
    inputs = [bytes(32), G.SQRT_ID_BYTES] + [rnd.randbytes(32) for _ in range(40)]
    for b in inputs:
        b = bytearray(b); b[0] &= 254; b[31] &= 127; b = bytes(b)
        P = L.map_to_curve_point(b)
        for Q in L.coset4(P):
            cands = L.map_to_curve_inverse(Q)
            assert b in cands
            for c in cands:
                if c is not None:
                    assert L.map_to_curve(c) == L.map_to_curve(b)


def test_constants_are_their_definitions(ho):
    p, d, i = L.p, H.d, H.SQRT_M1
    assert L.SQRT_ID ** 2 % p == i * d % p and L.SQRT_ID % 2 == 0
    assert L.DP1_OVER_DM1 * (d - 1) % p == (d + 1) % p
    assert L.MDOUBLE_INVSQRT_A_MINUS_D ** 2 * (-1 - d) % p == 4
    assert L.MIDOUBLE_INVSQRT_A_MINUS_D == L.MDOUBLE_INVSQRT_A_MINUS_D * i % p
    assert L.MINVSQRT_ONE_PLUS_D ** 2 * (1 + d) % p == 1
    for name, v in L.CONSTANTS.items():
        assert L.from_limbs51(L.STATED_LIMBS[name]) == v, name
        assert ho.constant(name) == v.to_bytes(32, "little"), name
    assert ho.constant("SQRT_M1") == i.to_bytes(32, "little") and ho.constant("MINUS_ONE") == (p - 1).to_bytes(32, "little")


def test_oracle_sha256(ho):
    rnd = random.Random(6)
    for n in list(range(0, 130)) + [1000]:
        m = rnd.randbytes(n)
        assert ho.sha256(m) == hashlib.sha256(m).digest()


def test_oracle_matches_every_vector():
    G.check_oracle(G.generate())


def test_oracle_matches_model_on_random_items(ho):
    rnd = random.Random(12)
    datas = [rnd.randbytes(16) for _ in range(300)]
    encs = ho.lizard_encode_batch(datas)
    assert encs == [L.lizard_encode(d) for d in datas]
    raw, st = ho.lizard_decode_batch(encs)
    assert st == bytes(300) and [raw[16 * i:16 * i + 16] for i in range(300)] == datas
    ins = [rnd.randbytes(32) for _ in range(300)]
    assert ho.map_to_curve_batch(ins) == [L.map_to_curve(b) for b in ins]
    pts = []
    for k in range(150):                              # Lizard points and random points, random representatives and Z
        enc = encs[k] if k % 2 else H.from_uniform_bytes(rnd.randbytes(64))
        Q = L.scale(L.coset4(L.ristretto_decode(enc))[rnd.randrange(4)], rnd.randrange(1, L.p))
        pts.append(Q)
    raw, masks = ho.map_to_curve_inverse_batch([L.limbs_bytes(Q) for Q in pts], lizard_oracle.FMT_EXTENDED)
    for i, Q in enumerate(pts):
        want = L.map_to_curve_inverse(Q)
        assert [raw[512 * i + 32 * j:512 * i + 32 * j + 32] for j in range(16)] == [x or bytes(32) for x in want]
        assert masks[i] == sum(1 << j for j, x in enumerate(want) if x is not None)
    raw, st = ho.lizard_decode_batch([L.limbs_bytes(Q) for Q in pts], lizard_oracle.FMT_EXTENDED)
    for i, Q in enumerate(pts):
        want = L.lizard_decode(Q)
        assert st[i] == (0 if want is not None else 1) and raw[16 * i:16 * i + 16] == (want or bytes(16))


def test_golden_labels(golden):
    g = json.loads(golden)
    labels = [v["label"] for v in g["points"]]
    assert sum("X = 0 or Y = 0" in lab for lab in labels) >= 4
    assert any("s = 0, t = 1" in lab for lab in labels) and any("s = 0, t = -1" in lab for lab in labels)
    assert sum("candidates reordered" in lab for lab in labels) >= 3
    assert sum(lab.startswith("undecodable") for lab in labels) >= 4
    assert any(0 < v["mask"] < 0xffff for v in g["points"]) and any(v["mask"] == 0 and v["status"] == 1 for v in g["points"])
    assert any(v["status"] == 1 and v["mask"] for v in g["points"])
    assert {v["label"] for v in g["e_inv_positive"]} == {"s = 0, t = 1", "s = 0, t = -1", "a square root exists", "no square root"}
