"""CPU checks of the hash-to-group fixtures: the golden file is what its generator writes, the model reproduces the
reference's known answers, the C oracle's constants are their definitions, and the C oracle equals the model on every
vector and on a few thousand random items of each kind."""
import json
import os
import random
import sys

import pytest

import h2c_model as M
import h2c_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_hash_to_curve_golden as G  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "hash_to_curve.json")) as f:
        return f.read()


@pytest.fixture(scope="module")
def ho():
    return h2c_oracle.load()


def test_file_is_what_the_generator_writes(golden):
    assert G.render(G.generate()) == golden


def test_model_reproduces_reference_kats():
    # generate() asserts each known answer against the model; repeat the headline ones explicitly
    g = G.generate()
    assert len(g["ristretto_elligator_sage"]) == 16 and len(g["one_way_map"]) == 11
    assert len(g["rfc9380_hash_to_curve"]) == 5 and len(g["rfc9380_encode_to_curve"]) == 5
    for v in g["one_way_map"]:
        assert M.from_uniform_bytes(bytes.fromhex(v["in"])).hex() == v["out"]
    for v in g["rfc9380_hash_to_curve"]:
        assert M.hash_to_curve(bytes.fromhex(v["msg"]), G.DST_RO).hex() == v["out"]


def test_golden_labels_and_survey(golden):
    g = json.loads(golden)
    labels = [v["label"] for v in g["from_uniform_edges"]]
    assert sum("D = 0" in lab for lab in labels) == 12
    assert any("Ns_D_is_sq true | false" in lab for lab in labels) and any("false | true" in lab for lab in labels)
    for h in g["d_zero_halves"]:
        assert M.map_inputs(int.from_bytes(bytes.fromhex(h), "little"))[1] == 0
    s = g["ns_d_is_sq_survey"]
    assert s["square"] + s["nonsquare"] == s["total"] == 1024 and min(s["square"], s["nonsquare"]) > 400
    assert {len(bytes.fromhex(v["dst"])) for v in g["xmd_boundaries"]} == {1, 45, 46, 124, 125, 255}
    assert any(v["exceptional"] for v in g["map_to_curve"])


def test_oracle_constants_are_their_definitions(ho):
    p, d = M.p, M.d
    want = {"ONE_MINUS_D_SQ": M.ONE_MINUS_D_SQ, "D_MINUS_ONE_SQ": M.D_MINUS_ONE_SQ, "SQRT_AD_MINUS_ONE": M.SQRT_AD_MINUS_ONE,
            "MINUS_ONE": p - 1, "MONTGOMERY_A": M.J, "MONTGOMERY_A_NEG": p - M.J, "SQRTAM2": M.SQRT_M486664,
            "ELL2_C2": 2 * pow(2, (p - 5) // 8, p) % p, "EDWARDS_D": d, "SQRT_M1": M.SQRT_M1}
    for name, v in want.items():
        assert ho.constant(name) == v.to_bytes(32, "little"), name
    assert M.SQRT_M486664 ** 2 % p == (-M.J - 2) % p
    c2 = want["ELL2_C2"]
    assert c2 * c2 % p in (2 * M.SQRT_M1 % p, (-2 * M.SQRT_M1) % p, 2, p - 2)


def test_oracle_matches_every_vector():
    G.check_oracle(G.generate())


def test_oracle_matches_model_on_random_items(ho):
    rnd = random.Random(11)
    for _ in range(2000):
        b = rnd.randbytes(64)
        assert ho.from_uniform_bytes(b) == M.from_uniform_bytes(b)
    msgs = [rnd.randbytes(rnd.randrange(0, 300)) for _ in range(2000)]
    assert ho.flat_batch("hash_from_bytes", msgs) == [M.hash_from_bytes(m) for m in msgs]
    for kind, fn in (("hash_to_curve", M.hash_to_curve), ("encode_to_curve", M.encode_to_curve)):
        dst = rnd.randbytes(rnd.randrange(1, 256))
        assert ho.flat_batch(kind, msgs, dst) == [fn(m, dst) for m in msgs], kind
