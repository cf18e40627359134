"""Write tests/golden/ed25519ph.json: Ed25519ph (RFC 8032 5.1, phflag = 1) vectors from a plain-Python model (hashlib and
tests/pyref.py), for ed25519-dalek's sign_prehashed / verify_prehashed / verify_prehashed_strict.

The file holds
  - the RFC 8032 7.3 vector (ed25519-dalek tests/ed25519.rs:104-146), which the model must reproduce;
  - seeded vectors with contexts of 0, 1, 6 ("edtest") and 255 bytes;
  - the cases of ed25519ph_sign_verify (tests/ed25519.rs:390-455): a good signature, the wrong prehash, and a signature
    over the other message;
  - a repudiation_prehash pair (tests/ed25519.rs:248-292) under the 8-torsion key EIGHT_TORSION[4] (order 2), found by a
    seeded search: one signature that passes verify_prehashed for two messages and fails verify_prehashed_strict.
Every vector records the model's verify / verify_strict codes (0 Ok, 1 Verify, 3 ScalarFormat, 4 PointDecompression).
With --check the generator also asserts that the C oracle (tests/ed25519ph_oracle.py) agrees with every vector.

    python tests/golden/make_ed25519ph_golden.py [--check]"""
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import pyref  # noqa: E402

OUT = os.path.join(HERE, "ed25519ph.json")
L = pyref.L
IDENTITY = (0, 1)
EIGHT_TORSION_4 = bytes([236] + [255] * 30 + [127])      # (0, -1), order 2 (u64/constants.rs EIGHT_TORSION[4])
RFC_SEED = "833fe62409237b9d62ec77587520911e9a759cec1d19755b7da901b96dca3d42"
RFC_PK = "ec172b93ad5e563bf4932c70e1245034c35467ef2efd4d64ebf819683467e2bf"
RFC_SIG = ("98a70222f0b8121aa9d30f813d683f809e462b469c7ff87639499bb94e6dae41"
           "31f85042463c2a355a2003d062adf5aaa10b8c61e636062aaad11c2a26083406")


def dom2(context):
    return b"SigEd25519 no Ed25519 collisions" + bytes([1, len(context)]) + context


def h_int(*parts):
    return int.from_bytes(hashlib.sha512(b"".join(parts)).digest(), "little")


def expand(seed):
    h = hashlib.sha512(seed).digest()
    a = bytearray(h[:32])
    a[0] &= 248; a[31] &= 127; a[31] |= 64
    return int.from_bytes(a, "little"), h[32:]


def public_key(seed):
    a, _ = expand(seed)
    return pyref.compress(pyref.mul(a, pyref.B))


def sign_prehashed(seed, ph, context=b""):
    a, prefix = expand(seed)
    A = pyref.compress(pyref.mul(a, pyref.B))
    r = h_int(dom2(context), prefix, ph) % L
    R = pyref.compress(pyref.mul(r, pyref.B))
    k = h_int(dom2(context), R, A, ph) % L
    return R + ((k * a + r) % L).to_bytes(32, "little")


def small_order(P):
    return pyref.mul(8, P) == IDENTITY


def verify_prehashed(ph, sig, pk, context=b"", strict=False):
    A = pyref.decompress(pk)
    if A is None:
        return 4
    s = int.from_bytes(sig[32:], "little")
    if s >= L:
        return 3
    if strict:
        R = pyref.decompress(sig[:32])
        if R is None or small_order(R) or small_order(A):
            return 1
    k = h_int(dom2(context), sig[:32], pk, ph) % L
    Rc = pyref.add(pyref.mul(s, pyref.B), pyref.neg(pyref.mul(k, A)))
    return 0 if pyref.compress(Rc) == sig[:32] else 1


def vector(label, seed, pk, ph, context, sig):
    return {"label": label, "seed": seed.hex() if seed else None, "pk": pk.hex(), "prehash": ph.hex(), "context": context.hex(),
            "sig": sig.hex(), "verify": verify_prehashed(ph, sig, pk, context),
            "verify_strict": verify_prehashed(ph, sig, pk, context, strict=True)}


def make():
    vs = []
    seed = bytes.fromhex(RFC_SEED)
    ph = hashlib.sha512(b"abc").digest()
    sig = sign_prehashed(seed, ph)
    assert public_key(seed).hex() == RFC_PK and sig.hex() == RFC_SIG, "the model does not reproduce RFC 8032 7.3"
    vs.append(vector("rfc8032_7.3", seed, public_key(seed), ph, b"", sig))
    rnd = random.Random(8032)
    for clen in (0, 1, 6, 255):
        for j in range(2):
            seed = rnd.randbytes(32)
            context = b"edtest" if clen == 6 else rnd.randbytes(clen)
            ph = hashlib.sha512(rnd.randbytes(rnd.randrange(200))).digest()
            vs.append(vector("context_%d_%d" % (clen, j), seed, public_key(seed), ph, context, sign_prehashed(seed, ph, context)))
    # ed25519ph_sign_verify
    seed = rnd.randbytes(32)
    pk = public_key(seed)
    context = b"testing testing 1 2 3"
    good, bad = hashlib.sha512(b"test message").digest(), hashlib.sha512(b"wrong message").digest()
    good_sig, bad_sig = sign_prehashed(seed, good, context), sign_prehashed(seed, bad, context)
    vs.append(vector("sign_verify_good", seed, pk, good, context, good_sig))
    vs.append(vector("sign_verify_bad_sig_on_good_prehash", seed, pk, good, context, bad_sig))
    vs.append(vector("sign_verify_good_sig_on_bad_prehash", seed, pk, bad, context, good_sig))
    # repudiation_prehash: R = sB - A with A = EIGHT_TORSION[4]; sB - kA == R iff k is odd for both messages
    A = pyref.decompress(EIGHT_TORSION_4)
    context = b"edtest"
    m1, m2 = hashlib.sha512(b"Send 100 USD to Alice").digest(), hashlib.sha512(b"Send 100000 USD to Alice").digest()
    srnd = random.Random(248)
    tries = 0
    while True:
        tries += 1
        s = srnd.randrange(1, L)
        R = pyref.compress(pyref.add(pyref.mul(s, pyref.B), pyref.neg(A)))
        if all(pyref.add(pyref.neg(A), pyref.mul(h_int(dom2(context), R, EIGHT_TORSION_4, m) % L, A)) == IDENTITY for m in (m1, m2)):
            break
    sig = R + s.to_bytes(32, "little")
    for label, m in (("repudiation_prehash_1", m1), ("repudiation_prehash_2", m2)):
        v = vector(label, None, EIGHT_TORSION_4, m, context, sig)
        assert v["verify"] == 0 and v["verify_strict"] == 1
        vs.append(v)
    assert [v["verify"] for v in vs[-5:-2]] == [0, 1, 1]
    return {"src": "tests/golden/make_ed25519ph_golden.py (RFC 8032 5.1; ed25519-dalek tests/ed25519.rs)",
            "repudiation_search_tries": tries, "vectors": vs}


def check_oracle(data):
    import ed25519ph_oracle
    o = ed25519ph_oracle.load()
    for v in data["vectors"]:
        ph, ctx, sig, pk = (bytes.fromhex(v[k]) for k in ("prehash", "context", "sig", "pk"))
        if v["seed"] and v["verify"] == 0:                 # the seed's own signature of this prehash
            assert o.sign_prehashed(bytes.fromhex(v["seed"]), ph, ctx) == (0, sig), v["label"]
        assert o.verify_prehashed(ph, sig, pk, ctx) == v["verify"], v["label"]
        assert o.verify_prehashed(ph, sig, pk, ctx, strict=True) == v["verify_strict"], v["label"]


if __name__ == "__main__":
    data = make()
    if "--check" in sys.argv:
        check_oracle(data)
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote %s (%d vectors)" % (OUT, len(data["vectors"])))
