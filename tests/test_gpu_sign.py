"""GPU Ed25519 signing and Ed25519ph: ed25519_b200_verifying_keys / sign_flat / sign_prehashed / verify_prehashed_each
against TESTVECTORS, the Ed25519ph fixture, the C oracles and `cryptography`, at piece boundaries and at every SHA-512
block boundary of both hashes."""
import ctypes as C
import hashlib
import json
import os
import random

import numpy as np
import pytest

import ed25519ph_oracle
import oracle_lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, VERIFY, SCALARFMT, POINTDEC, CTXLEN, INVALID = 0, 1, 3, 4, 5, -1
EIGHT_TORSION_4 = bytes([236] + [255] * 30 + [127])


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def pho():
    return ed25519ph_oracle.load()


@pytest.fixture(scope="module")
def ph_golden():
    with open(os.path.join(ROOT, "tests", "golden", "ed25519ph.json")) as f:
        return json.load(f)["vectors"]


def flat(msgs):
    offs = np.zeros(len(msgs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m) for m in msgs]) if msgs else []
    return np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy(), offs


def split(raw, k):
    return [raw[k * i:k * i + k] for i in range(len(raw) // k)]


def sign(eng, seeds, msgs):
    fl, offs = flat(msgs)
    return split(eng.sign_flat(b"".join(seeds), len(seeds), fl, offs, len(msgs)), 64)


def verify_each(eng, msgs, sigs, keys, strict):
    fl, offs = flat(msgs)
    return eng.verify_each_flat(fl, offs, b"".join(sigs), b"".join(keys), len(msgs), strict=strict)


def test_testvectors(eng):
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_testvectors.json")) as f:
        tv = json.load(f)["vectors"]
    seeds = [bytes.fromhex(v["seed"]) for v in tv]
    msgs = [bytes.fromhex(v["msg"]) for v in tv]
    assert split(eng.verifying_keys(b"".join(seeds), len(seeds)), 32) == [bytes.fromhex(v["pk"]) for v in tv]
    assert sign(eng, seeds, msgs) == [bytes.fromhex(v["sig"]) for v in tv]
    for s, m, v in zip(seeds, msgs, tv):                  # one key for the whole (one-message) batch
        fl, offs = flat([m])
        assert eng.sign_flat(s, 1, fl, offs, 1) == bytes.fromhex(v["sig"])


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, (1 << 16) - 1, (1 << 16) + 1, (1 << 17) + 3])
@pytest.mark.parametrize("one_key", [False, True])
def test_random_batches(eng, orc, n, one_key):
    rnd = random.Random(n * 2 + one_key)
    seeds = [rnd.randbytes(32) for _ in range(1 if one_key else n)]
    msgs = [rnd.randbytes(rnd.randrange(0, 100)) for _ in range(n)]
    fl, offs = flat(msgs)
    sigs = split(eng.sign_flat(b"".join(seeds), len(seeds) if n else 0, fl, offs, n), 64)
    assert len(sigs) == n
    if not n:
        return
    keys = [orc.public_key(s) for s in seeds] if n <= 4096 or one_key else None
    idx = range(n) if n <= 4096 else sorted(rnd.sample(range(n), 4096))
    if keys is None:
        pk_all = split(eng.verifying_keys(b"".join(seeds), n), 32)
        for i in idx[:256]:
            assert pk_all[i] == orc.public_key(seeds[i])
    else:
        pk_all = keys * n if one_key else keys
    for i in idx:
        seed = seeds[0 if one_key else i]
        assert sigs[i] == orc.sign(msgs[i], seed), i
    for strict in (False, True):
        rc, res = eng.verify_each_flat(fl, offs, b"".join(sigs), b"".join(pk_all), n, strict=strict)
        assert rc == OK and not any(res)


def test_message_lengths_at_block_boundaries(eng, orc):
    rnd = random.Random(5)
    lens = [0, 47, 48, 79, 80, 175, 176, 207, 208, 111, 112, 239, 240, 1 << 20, 3, 128, 255, 256]
    msgs = [rnd.randbytes(k) for k in lens]
    for one_key in (False, True):
        seeds = [rnd.randbytes(32)] if one_key else [rnd.randbytes(32) for _ in msgs]
        sigs = sign(eng, seeds, msgs)
        for i, m in enumerate(msgs):
            assert sigs[i] == orc.sign(m, seeds[0 if one_key else i]), lens[i]


def test_ph_fixture_sign_and_verify(eng, pho, ph_golden):
    for v in ph_golden:
        ph, ctx, sig, pk = (bytes.fromhex(v[k]) for k in ("prehash", "context", "sig", "pk"))
        if v["seed"] and v["verify"] == OK:
            rc, got = eng.sign_prehashed(bytes.fromhex(v["seed"]), 1, ph, 1, ctx)
            assert rc == OK and got == sig, v["label"]
    phs = b"".join(bytes.fromhex(v["prehash"]) for v in ph_golden)
    sigs = b"".join(bytes.fromhex(v["sig"]) for v in ph_golden)
    keys = b"".join(bytes.fromhex(v["pk"]) for v in ph_golden)
    for each_comb in (0, 2, 1):
        eng.set_option("each_comb", each_comb)
        for v in ph_golden:                                # one context per call
            ctx = bytes.fromhex(v["context"])
            for strict in (False, True):
                _, res = eng.verify_prehashed_each(bytes.fromhex(v["prehash"]), bytes.fromhex(v["sig"]), bytes.fromhex(v["pk"]), 1,
                                                   ctx, strict)
                assert res == [v["verify_strict" if strict else "verify"]], (v["label"], each_comb, strict)
        # a whole batch under the RFC's empty context: the vectors signed under another context fail, in both paths
        for strict in (False, True):
            _, res = eng.verify_prehashed_each(phs, sigs, keys, len(ph_golden), b"", strict)
            want = [pho.verify_prehashed(bytes.fromhex(v["prehash"]), bytes.fromhex(v["sig"]), bytes.fromhex(v["pk"]), b"", strict)
                    for v in ph_golden]
            assert res == want
    eng.set_option("each_comb", 1)


def test_ph_block_boundaries_of_the_context(eng, pho):
    """Contexts at which the nonce hash dom2 || prefix || PH and the challenge hash dom2 || R || A || PH gain a block."""
    rnd = random.Random(6)
    seed = rnd.randbytes(32)
    pk = oracle_lib.load().public_key(seed)
    # |dom2 || prefix || PH| + 17 = 147 + |C| crosses 256 and 384 at |C| = 110 / 238; |dom2 || R || A || PH| + 17 at 78 / 206
    for clen in [0, 1, 6, 7, 8, 9, 15, 16, 17, 18, 45, 46, 47, 48, 49, 77, 78, 79, 80, 81, 109, 110, 111, 112, 113, 200, 205,
                 206, 207, 208, 209, 237, 238, 239, 254, 255]:
        ctx = rnd.randbytes(clen)
        phs = [rnd.randbytes(64) for _ in range(3)]
        rc, raw = eng.sign_prehashed(seed, 1, b"".join(phs), 3, ctx)
        assert rc == OK
        for ph, sig in zip(phs, split(raw, 64)):
            assert (0, sig) == pho.sign_prehashed(seed, ph, ctx), clen
        rc, res = eng.verify_prehashed_each(b"".join(phs), raw, pk * 3, 3, ctx, True)
        assert rc == OK and res == [OK] * 3


@pytest.mark.parametrize("nkeys", [61, None])
def test_ph_large_batch(eng, pho, nkeys):
    """2^17 + 3 Ed25519ph signatures by 61 keys (per-key comb path) and by distinct keys (plain path), with failures."""
    n = (1 << 17) + 3
    rnd = random.Random(7 if nkeys else 8)
    gen = np.random.Generator(np.random.PCG64(9))
    k = nkeys or n
    seeds = gen.integers(0, 256, size=(k, 32), dtype=np.uint8)
    pks = np.frombuffer(eng.verifying_keys(seeds, k), dtype=np.uint8).reshape(k, 32)
    phs = gen.integers(0, 256, size=(n, 64), dtype=np.uint8)
    ctx = b"bulk"
    key_of = np.arange(n) % k
    sigs = np.empty((n, 64), dtype=np.uint8)
    if nkeys:
        for j in range(k):                                 # one signing call per key (n_seeds = 1)
            sel = np.nonzero(key_of == j)[0]
            rc, raw = eng.sign_prehashed(seeds[j].tobytes(), 1, np.ascontiguousarray(phs[sel]), len(sel), ctx)
            assert rc == OK
            sigs[sel] = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 64)
    else:
        rc, raw = eng.sign_prehashed(seeds, n, phs, n, ctx)
        assert rc == OK
        sigs[:] = np.frombuffer(raw, dtype=np.uint8).reshape(n, 64)
    keys = np.ascontiguousarray(pks[key_of])
    for i in sorted(rnd.sample(range(n), 512)):
        assert pho.sign_prehashed(seeds[key_of[i]].tobytes(), phs[i].tobytes(), ctx) == (0, sigs[i].tobytes())
    bad = [5, 65535, 65536, n - 1]
    for i in bad:
        sigs[i, 3] ^= 1
    for strict in (False, True):
        rc, res = eng.verify_prehashed_each(phs, sigs, keys, n, ctx, strict)
        assert rc == VERIFY and [i for i, r in enumerate(res) if r] == bad


def test_ph_error_kinds_and_precedence(eng, pho, ph_golden):
    rnd = random.Random(10)
    ctx = b"edtest"
    seeds = [rnd.randbytes(32) for _ in range(64)]
    keys = [oracle_lib.load().public_key(s) for s in seeds]
    phs = [rnd.randbytes(64) for _ in range(64)]
    sigs = [eng.sign_prehashed(s, 1, p, 1, ctx)[1] for s, p in zip(seeds, phs)]
    s, k, p = list(sigs), list(keys), list(phs)
    p[3] = bytes(64)                                                            # Verify
    x = bytearray(s[10]); x[63] |= 0xf0; s[10] = bytes(x)                       # ScalarFormat
    k[20] = (2).to_bytes(32, "little")                                          # PointDecompression
    x = bytearray(s[30]); x[63] |= 0xf0; s[30] = bytes(x); k[30] = (2).to_bytes(32, "little")   # the key first
    s[40] = (2).to_bytes(32, "little") + s[40][32:]                             # undecodable R
    x = bytearray(s[50]); x[0] ^= 1; s[50] = bytes(x)                           # wrong R
    rep = [v for v in ph_golden if v["label"].startswith("repudiation")][0]     # small-order key: strict rejects
    p[60], s[60], k[60] = (bytes.fromhex(rep[f]) for f in ("prehash", "sig", "pk"))
    for each_comb in (0, 2):
        eng.set_option("each_comb", each_comb)
        for strict in (False, True):
            rc, res = eng.verify_prehashed_each(b"".join(p), b"".join(s), b"".join(k), 64, ctx, strict)
            want = [pho.verify_prehashed(p[i], s[i], k[i], ctx, strict) for i in range(64)]
            assert res == want and rc == VERIFY
            assert (res[3], res[10], res[20], res[30], res[40], res[50]) == (VERIFY, SCALARFMT, POINTDEC, POINTDEC, VERIFY, VERIFY)
            assert res[60] == (VERIFY if strict else OK)
    eng.set_option("each_comb", 1)


def test_context_length_and_domain_separation(eng, orc):
    seed = bytes(range(32))
    pk = orc.public_key(seed)
    ph = hashlib.sha512(b"message").digest()
    assert eng.sign_prehashed(seed, 1, ph, 1, bytes(256))[0] == CTXLEN
    assert eng.sign_prehashed(seed, 1, ph, 1, bytes(255))[0] == OK
    with pytest.raises(Exception):
        eng.verify_prehashed_each(ph, bytes(64), pk, 1, bytes(256))
    assert eng.lib.ed25519_b200_verify_prehashed_each(eng.h, ph, None, 256, bytes(64), pk, 1, 0, (C.c_uint8 * 1)()) == INVALID
    _, sig_ph = eng.sign_prehashed(seed, 1, ph, 1, b"C")
    assert eng.verify_prehashed_each(ph, sig_ph, pk, 1, b"C")[1] == [OK]
    assert eng.verify_prehashed_each(ph, sig_ph, pk, 1, b"D")[1] == [VERIFY]              # context C signs nothing under C'
    assert verify_each(eng, [ph], [sig_ph], [pk], False)[1] == [VERIFY]                   # Ed25519ph is not pure Ed25519
    sig_pure = sign(eng, [seed], [ph])[0]
    assert eng.verify_prehashed_each(ph, sig_pure, pk, 1, b"")[1] == [VERIFY]             # nor the other way round
    assert eng.verify_prehashed_each(ph, sig_pure, pk, 1, None)[1] == [VERIFY]


def test_sign_batch_flat_compatibility(eng, orc):
    ed = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.ed25519")
    rnd = random.Random(11)
    n = 300
    seeds = [rnd.randbytes(32) for _ in range(n)]
    msgs = [rnd.randbytes(rnd.randrange(300)) for _ in range(n)]
    fl, offs = flat(msgs)
    pks, sigs = eng.sign_batch_flat(b"".join(seeds), fl, offs, n)
    assert pks == eng.verifying_keys(b"".join(seeds), n)
    assert sigs == eng.sign_flat(b"".join(seeds), n, fl, offs, n)
    for i in range(0, n, 7):
        assert split(sigs, 64)[i] == ed.Ed25519PrivateKey.from_private_bytes(seeds[i]).sign(msgs[i])


def test_argument_checks(eng):
    lib, h = eng.lib, eng.h
    seeds, fl = bytes(96), np.zeros(8, dtype=np.uint8)
    offs = np.array([0, 1, 2, 3], dtype=np.uint64)
    out = (C.c_uint8 * 256)()
    ph = bytes(192)
    sf = lib.ed25519_b200_sign_flat
    assert sf(h, seeds, 2, fl.ctypes.data, offs.ctypes.data, 3, out) == INVALID               # n_seeds not in {1, n}
    assert sf(h, seeds, 0, fl.ctypes.data, offs.ctypes.data, 3, out) == INVALID
    assert sf(h, seeds, 3, fl.ctypes.data, offs.ctypes.data, 3, out) == OK
    assert sf(h, seeds, 1, fl.ctypes.data, offs.ctypes.data, 3, out) == OK
    assert sf(h, None, 3, fl.ctypes.data, offs.ctypes.data, 3, out) == INVALID
    assert sf(h, seeds, 3, fl.ctypes.data, offs.ctypes.data, 3, None) == INVALID
    assert sf(h, seeds, 3, None, offs.ctypes.data, 3, out) == INVALID                       # non-empty messages need a buffer
    assert sf(h, seeds, 3, fl.ctypes.data, None, 3, out) == INVALID
    bad = np.array([1, 1, 2, 3], dtype=np.uint64)
    assert sf(h, seeds, 3, fl.ctypes.data, bad.ctypes.data, 3, out) == INVALID               # offsets[0] != 0
    bad = np.array([0, 2, 1, 3], dtype=np.uint64)
    assert sf(h, seeds, 3, fl.ctypes.data, bad.ctypes.data, 3, out) == INVALID               # decreasing
    zero = np.zeros(4, dtype=np.uint64)
    assert sf(h, seeds, 3, None, zero.ctypes.data, 3, out) == OK                            # all empty: no buffer needed
    assert sf(h, None, 0, None, None, 0, None) == OK                                        # n = 0
    sp = lib.ed25519_b200_sign_prehashed
    assert sp(h, seeds, 3, ph, 3, None, 1, out) == INVALID                                  # NULL context, non-zero length
    assert sp(h, seeds, 3, None, 3, None, 0, out) == INVALID
    assert sp(h, seeds, 2, ph, 3, None, 0, out) == INVALID
    assert sp(h, seeds, 3, ph, 3, None, 0, out) == OK
    assert lib.ed25519_b200_verifying_keys(h, None, 1, out) == INVALID
    assert lib.ed25519_b200_verifying_keys(h, None, 0, None) == OK
    vp = lib.ed25519_b200_verify_prehashed_each
    assert vp(h, ph, None, 1, bytes(64), bytes(32), 1, 0, out) == INVALID
    assert vp(h, None, None, 0, bytes(64), bytes(32), 1, 0, out) == INVALID
    assert vp(h, None, None, 0, None, None, 0, 0, None) == OK


def test_python_functions(eng, orc, pho):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(12)
    seeds = [rnd.randbytes(32) for _ in range(3)]
    msgs = [b"", b"abc", rnd.randbytes(500)]
    assert pkg.ed25519_verifying_keys(seeds[0], engine=eng) == orc.public_key(seeds[0])
    assert pkg.ed25519_verifying_keys(seeds, engine=eng) == [orc.public_key(s) for s in seeds]
    assert pkg.ed25519_sign(seeds[0], b"abc", engine=eng) == orc.sign(b"abc", seeds[0])
    assert pkg.ed25519_sign(seeds[0], msgs, engine=eng) == [orc.sign(m, seeds[0]) for m in msgs]
    assert pkg.ed25519_sign(seeds, msgs, engine=eng) == [orc.sign(m, s) for m, s in zip(msgs, seeds)]
    assert pkg.ed25519_sign(seeds[0], [], engine=eng) == []
    hs = [hashlib.sha512(m) for m in msgs]
    sig1 = pkg.ed25519_sign_prehashed(seeds[1], hs[1], b"ctx", engine=eng)
    assert (0, sig1) == pho.sign_prehashed(seeds[1], hs[1].digest(), b"ctx")
    sigs = pkg.ed25519_sign_prehashed(seeds, [h.digest() for h in hs], engine=eng)
    assert sigs == pkg.ed25519_sign_prehashed(seeds, hs, context=None, engine=eng)
    pks = [orc.public_key(s) for s in seeds]
    assert pkg.ed25519_verify_prehashed(hs, sigs, pks, engine=eng) == [0, 0, 0]
    assert pkg.ed25519_verify_prehashed(hs, sigs, pks, strict=True, engine=eng) == [0, 0, 0]
    assert pkg.ed25519_verify_prehashed(hs[1], sig1, pks[1], context=b"ctx", engine=eng) == 0
    assert pkg.ed25519_verify_prehashed(hs[1], sig1, pks[1], context=b"ctz", engine=eng) == 1
    with pytest.raises(pkg.SignatureError) as e:
        pkg.ed25519_sign_prehashed(seeds[0], hs[0], bytes(256), engine=eng)
    assert e.value.code == 5 and e.value.kind == "PrehashedContextLength"
    with pytest.raises(ValueError):
        pkg.ed25519_verify_prehashed(hs[0], sig1, pks[0], context=bytes(256), engine=eng)
    with pytest.raises(ValueError):
        pkg.ed25519_sign(seeds[:2], msgs, engine=eng)
