"""tests/golden/ristretto.json against its generator, the big-integer decode and the C oracle (CPU only).

The GPU tests feed these vectors to every Ristretto decode site; what makes them worth feeding is checked here:
each label is what CompressedRistretto::decompress (ristretto.rs:266-345) computes, the oracle agrees with it, and
every rejection term fires alone in enough vectors that a decoder missing that term is caught."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_ristretto_golden as gen  # noqa: E402


@pytest.fixture(scope="module")
def doc():
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        return json.load(f)


def vectors(doc):
    return [(name, bytes.fromhex(v["s"]), v["terms"]) for name, vs in doc["classes"].items() for v in vs]


def test_file_is_what_the_generator_writes(doc):
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        assert f.read() == gen.render(gen.build_doc())


def test_labels_are_the_decode_terms(doc):
    assert doc["terms"] == gen.TERMS
    for name, enc, terms in vectors(doc):
        assert gen.decode_terms(enc) == terms, (name, enc.hex())
        assert (name == "valid") == (terms == []), (name, enc.hex())
        assert name == "valid" or name in terms, (name, enc.hex())


def test_oracle_rejects_exactly_the_labelled_vectors(oracle, doc):
    for name, enc, terms in vectors(doc):
        P = oracle.ristretto_decompress(enc)
        assert (P is None) == bool(terms), (name, enc.hex(), terms)
        if P is not None:
            assert oracle.ristretto_compress(P) == enc, (name, enc.hex())


def test_every_term_fires_alone(doc):
    """16 single-term vectors per class; y = 0 alone happens only for s = p - 1"""
    for term in gen.TERMS:
        singles = [v["s"] for v in doc["classes"][term] if v["terms"] == [term]]
        assert len(singles) >= (1 if term == "y_zero" else gen.SINGLES), term
    assert [v["s"] for v in doc["classes"]["y_zero"] if v["terms"] == ["y_zero"]] == [gen.b32(gen.P - 1).hex()]
    noncanon = {int.from_bytes(bytes.fromhex(v["s"]), "little") for v in doc["classes"]["noncanonical"]}
    assert set(range(gen.P, 2**255)) <= noncanon
    assert [v["terms"] for v in doc["classes"]["noncanonical"] if v["s"] == gen.b32(gen.P).hex()] == [["noncanonical"]]


def test_decode_model_on_known_points(oracle, kat):
    """the model accepts the reference's small multiples and random encodings, and rejects what it must"""
    import random
    rnd = random.Random(9)
    B = oracle.basepoint()
    for h in kat["ristretto"]["SMALL_MULTIPLES"]["hex"]:
        assert gen.decode_terms(bytes.fromhex(h)) == []
    for _ in range(32):
        enc = oracle.ristretto_compress(oracle.scalarmul(rnd.randrange(gen.P).to_bytes(32, "little")[:31] + b"\0", B))
        assert gen.decode_terms(enc) == []
        neg = gen.b32(gen.P - int.from_bytes(enc, "little")) if enc != bytes(32) else None
        if neg is not None:
            assert gen.decode_terms(neg) == ["negative"]
    assert gen.decode_terms(b"\xff" * 32)[0] == "noncanonical"
