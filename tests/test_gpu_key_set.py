"""GPU tests of resident verifying-key sets: ed25519_b200_key_set_new / _verify_flat / _verify_flat_dev /
_verify_prehashed and VerifyingKeySet.  A set decompresses and tabulates its keys once (VerifyingKey::from_bytes,
E/verifying.rs:167-175) and then verifies signatures under key indices; every verdict must equal the per-signature
verifier's (ed25519_b200_verify_each_flat / verify_prehashed_each) on the same inputs with the key bytes inlined, and the
oracle's."""
import ctypes as C
import hashlib
import json
import os
import random
import threading

import numpy as np
import pytest

import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = bytes.fromhex
OK, VERIFY, SCALARFMT, POINTDEC = 0, 1, 3, 4
INVALID = -1


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def vectors():
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_validation.json")) as f:
        vec = json.load(f)["vectors"]
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_testvectors.json")) as f:
        tv = json.load(f)["vectors"]
    msgs = [v["msg"].encode() for v in vec] + [H(v["msg"]) for v in tv]
    sigs = [H(v["sig"]) for v in vec] + [H(v["sig"]) for v in tv]
    keys = [H(v["key"]) for v in vec] + [H(v["pk"]) for v in tv]
    return msgs, sigs, keys


def flat(msgs):
    offs = np.zeros(len(msgs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy(), offs


def u32(xs):
    return np.ascontiguousarray(np.asarray(xs, dtype=np.uint32))


class KeySet:
    """A set made through the Engine methods, with its key bytes kept for the inlined comparisons."""

    def __init__(self, eng, keys):
        self.eng, self.keys = eng, list(keys)
        rc, self.h, self.ok, self.weak = eng.key_set_new(b"".join(self.keys), len(self.keys))
        assert rc == OK and self.h is not None and self.ok == b"\x01" * len(self.keys)

    def close(self):
        self.eng.key_set_destroy(self.h)

    def verify(self, msgs, sigs, idx, strict=False, device=False):
        n = len(sigs)
        fl, offs = flat(msgs)
        ib = u32(idx) if idx is not None else None
        if not device:
            return self.eng.key_set_verify_flat(self.h, fl, offs, b"".join(sigs), ib, n, strict)
        import torch
        dev = torch.device("cuda", 0)
        d = [torch.from_numpy(x).to(dev) for x in (fl, offs.view(np.int64), np.frombuffer(b"".join(sigs) or bytes(64), dtype=np.uint8).copy())]
        di = torch.from_numpy(ib.view(np.int32)).to(dev) if ib is not None else None
        return self.eng.key_set_verify_flat(self.h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                            di.data_ptr() if di is not None else None, n, strict, device_ptrs=True)

    def inline(self, idx, n):
        return [self.keys[idx[i] if idx is not None else 0] for i in range(n)]


def each(eng, msgs, sigs, keys, strict):
    fl, offs = flat(msgs)
    return eng.verify_each_flat(fl, offs, b"".join(sigs), b"".join(keys), len(sigs), strict=strict)


# ---- 1. the reference's vectors ------------------------------------------------------------------------------------
@pytest.mark.parametrize("strict", [False, True])
def test_vector_parity(eng, oracle, vectors, strict):
    """All 914 VALIDATIONVECTORS and 128 TESTVECTORS through a set of their distinct decodable keys: the non-canonical
    keys among them check that the set hashes the bytes it was given."""
    msgs, sigs, keys = vectors
    decodable = [k for k in dict.fromkeys(keys) if oracle.decompress(k) is not None]
    assert any(oracle.compress(oracle.decompress(k)) != k for k in decodable)   # non-canonical A encodings
    pos = {k: i for i, k in enumerate(decodable)}
    use = [i for i, k in enumerate(keys) if k in pos]
    m, s, idx = [msgs[i] for i in use], [sigs[i] for i in use], [pos[keys[i]] for i in use]
    ks = KeySet(eng, decodable)
    try:
        for device in (False, True):
            rc, res = ks.verify(m, s, idx, strict, device=device)
            rc_e, want = each(eng, m, s, ks.inline(idx, len(s)), strict)
            assert res == want and rc == rc_e, device
        assert res == [oracle.verify(mm, ss, keys[i], strict=strict) for mm, ss, i in zip(m, s, use)]
        assert POINTDEC not in res
    finally:
        ks.close()


def test_undecodable_keys_fail_new(eng, oracle, vectors):
    """the vectors' keys with encodings that do not decode (y with no x, canonical and not) spread among them"""
    _, _, keys = vectors
    distinct = [k for k in dict.fromkeys(keys) if oracle.decompress(k) is not None]
    cands = [y.to_bytes(32, "little") for y in list(range(2, 64)) + [pyref.p + y for y in range(2, 19)]]
    undecodable = [e for e in cands if oracle.decompress(e) is None][:6]
    assert len(undecodable) == 6
    for j, e in enumerate(undecodable):
        distinct.insert(37 * j + 5, e)
    bad = [i for i, k in enumerate(distinct) if k in undecodable]
    assert len(bad) == 6
    rc, h, ok, weak = eng.key_set_new(b"".join(distinct), len(distinct))
    assert rc == POINTDEC and h is None
    assert [i for i, b in enumerate(ok) if not b] == bad
    import curve25519_dalek_b200 as pkg
    with pytest.raises(pkg.SignatureError) as e:
        pkg.VerifyingKeySet(distinct, engine=eng)
    assert e.value.kind == "PointDecompression" and ("key %d " % bad[0]) in str(e.value)


# ---- 2. error kinds ------------------------------------------------------------------------------------------------
def test_error_kinds(eng, oracle):
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_testvectors.json")) as f:
        tv = json.load(f)["vectors"]
    m = [H(v["msg"]) for v in tv]
    s = [H(v["sig"]) for v in tv]
    keys = [H(v["pk"]) for v in tv]
    ks = KeySet(eng, keys)
    idx = list(range(len(tv)))
    try:
        for strict in (False, True):
            assert ks.verify(m, s, idx, strict) == (OK, [OK] * len(tv))
        m[3] = m[3] + b"x"                                                    # Verify
        x = bytearray(s[10]); x[63] |= 0xf0; s[10] = bytes(x)                 # s >= l: ScalarFormat
        s[40] = (2).to_bytes(32, "little") + s[40][32:]                       # undecodable R: Verify
        x = bytearray(s[50]); x[0] ^= 1; s[50] = bytes(x)                     # wrong R
        x = bytearray(s[60]); x[63] |= 0xf0; s[60] = (2).to_bytes(32, "little") + bytes(x[32:])   # both: ScalarFormat first
        T = torsion_points(oracle)[3]                                         # order 2
        small_r = oracle.compress(T) + s[70][32:]                             # strict: R of small order
        s[70] = small_r
        for strict in (False, True):
            rc, res = ks.verify(m, s, idx, strict)
            want = [oracle.verify(m[i], s[i], keys[i], strict=strict) for i in range(len(tv))]
            assert res == want and rc == VERIFY
            assert res == each(eng, m, s, keys, strict)[1]
            assert [i for i, r in enumerate(res) if r] == [3, 10, 40, 50, 60, 70]
            assert (res[10], res[60]) == (SCALARFMT, SCALARFMT)
    finally:
        ks.close()


def test_strict_small_order_r(eng, oracle):
    """R of small order with s = k a: R' = [s]B - [k]A is the identity, so verify accepts R = the identity and
    verify_strict rejects it, as the per-signature verifier does."""
    rnd = random.Random(5)
    seed = rnd.randbytes(32)
    A = oracle.public_key(seed)
    a = int.from_bytes(hashlib.sha512(seed).digest()[:32], "little")
    a = (a & ~7 & ((1 << 254) - 1)) | (1 << 254)                     # clamp_integer (C/scalar.rs:1407-1412)
    msgs, sigs = [], []
    for t in [oracle.identity()] + torsion_points(oracle):
        R = oracle.compress(t)
        for j in range(4):
            msg = b"small R %d" % j
            k = int.from_bytes(hashlib.sha512(R + A + msg).digest(), "little") % pyref.L
            msgs.append(msg); sigs.append(R + ((k * a) % pyref.L).to_bytes(32, "little"))
    ks = KeySet(eng, [A])
    try:
        for strict in (False, True):
            rc, res = ks.verify(msgs, sigs, None, strict)
            assert res == [oracle.verify(mm, ss, A, strict=strict) for mm, ss in zip(msgs, sigs)]
            assert res == each(eng, msgs, sigs, [A] * len(sigs), strict)[1]
        assert all(r == VERIFY for r in res)                     # strict
        assert ks.verify(msgs, sigs, None, False)[1][:4] == [OK] * 4     # R = the identity passes verify
    finally:
        ks.close()


# ---- 3. weak keys --------------------------------------------------------------------------------------------------
def _torsion_encodings(oracle):
    encs = [oracle.compress(oracle.identity())] + [oracle.compress(t) for t in torsion_points(oracle)]
    p = pyref.p
    extra = [(p + 1).to_bytes(32, "little"),                                   # y = 1, non-canonical
             p.to_bytes(32, "little"),                                         # y = 0, non-canonical
             (p | (1 << 255)).to_bytes(32, "little"),                          # and its sign bit
             (1 | (1 << 255)).to_bytes(32, "little"),                          # y = 1, sign bit set ("-0")
             ((p - 1) | (1 << 255)).to_bytes(32, "little")]                    # y = -1, sign bit set
    return encs, [e for e in extra if oracle.decompress(e) is not None]


def test_weak_keys(eng, oracle):
    canon, noncanon = _torsion_encodings(oracle)
    assert len(canon) == 8 and len(set(canon)) == 8 and noncanon
    rnd = random.Random(3)
    rand = [oracle.public_key(rnd.randbytes(32)) for _ in range(16)]
    keys = canon + noncanon + rand
    want = [int(oracle.is_identity(oracle.mul_by_pow_2(oracle.decompress(k), 3))) for k in keys]
    assert want == [1] * (len(canon) + len(noncanon)) + [0] * len(rand)
    ks = KeySet(eng, keys)
    try:
        assert list(ks.weak) == want
        # R = rB, s = r: valid under verify for any encoding of the identity (k A = identity); every weak key fails
        # strict, every result equals the per-signature verifier's
        msgs, sigs, idx = [], [], []
        for i in range(len(keys)):
            for j in range(3):
                r = rnd.randrange(pyref.L)
                R = oracle.compress(oracle.scalarmul(r.to_bytes(32, "little"), oracle.basepoint()))
                msgs.append(b"weak %d %d" % (i, j)); sigs.append(R + r.to_bytes(32, "little")); idx.append(i)
        for strict in (False, True):
            rc, res = ks.verify(msgs, sigs, idx, strict)
            assert res == each(eng, msgs, sigs, ks.inline(idx, len(sigs)), strict)[1]
            assert res == [oracle.verify(mm, ss, keys[t], strict=strict) for mm, ss, t in zip(msgs, sigs, idx)]
            if strict:
                assert all(res[q] == VERIFY for q in range(len(idx)) if want[idx[q]])
        ident = [q for q in range(len(idx)) if oracle.is_identity(oracle.decompress(keys[idx[q]]))]
        assert len(ident) >= 3 and all(ks.verify(msgs, sigs, idx, False)[1][q] == OK for q in ident)
    finally:
        ks.close()
    import curve25519_dalek_b200 as pkg
    s = pkg.VerifyingKeySet(keys, engine=eng)
    assert [s.is_weak(i) for i in range(len(keys))] == [bool(w) for w in want] and len(s) == len(keys)
    s.close()


# ---- 4. indices and sizes ------------------------------------------------------------------------------------------
def _signed(eng, k, n, seed, lens_mod=7):
    """k keys from seeds, n signatures with random key indices, some corrupted: (key bytes, msgs flat, offs, sigs,
    pubkeys per signature, indices)."""
    g = np.random.Generator(np.random.PCG64(seed))
    kseeds = g.integers(0, 256, size=(k, 32), dtype=np.uint8)
    keys = eng.verifying_keys(kseeds, k)
    idx = u32(g.integers(0, k, size=n)) if n else u32([])
    lens = (np.arange(n) % lens_mod) * 11
    offs = np.zeros(n + 1, dtype=np.uint64); offs[1:] = np.cumsum(lens)
    fl = g.integers(0, 256, size=int(offs[-1]) + 1, dtype=np.uint8)
    if n:
        pks, sigs = eng.sign_batch_flat(np.ascontiguousarray(kseeds[idx]), fl, offs, n)
    else:
        pks, sigs = b"", b""
    sg = np.frombuffer(sigs, dtype=np.uint8).copy()
    for i in sorted(set(g.integers(0, max(n, 1), size=min(n, 7)).tolist())):
        sg[64 * i + 5 + (i % 50)] ^= 4
    return keys, fl, offs, sg, pks, idx


def _check(eng, h, fl, offs, sg, pks, idx, n, strict=False, device=False):
    rc_e, want = eng.verify_each_flat(fl, offs, sg, pks, n, strict=strict)
    if device:
        import torch
        dev = torch.device("cuda", 0)
        d = [torch.from_numpy(x).to(dev) for x in (fl, offs.view(np.int64), sg if n else np.zeros(64, np.uint8))]
        di = torch.from_numpy(idx.view(np.int32) if n else np.zeros(1, np.int32)).to(dev) if idx is not None else None
        rc, res = eng.key_set_verify_flat(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                          di.data_ptr() if di is not None else None, n, strict, device_ptrs=True)
    else:
        rc, res = eng.key_set_verify_flat(h, fl, offs, sg, idx, n, strict)
    assert rc == rc_e and res == want
    return res


def test_null_indices_mean_key_zero(eng):
    keys, fl, offs, sg, pks, _ = _signed(eng, 1, 300, 11)
    rc, h, _, _ = eng.key_set_new(keys, 1)
    try:
        for device in (False, True):
            res = _check(eng, h, fl, offs, sg, pks, None, 300, device=device)
            assert 0 < sum(1 for r in res if r) <= 7
    finally:
        eng.key_set_destroy(h)
    # a set of three keys with indices NULL verifies everything under key 0
    keys3, fl, offs, sg, _, _ = _signed(eng, 3, 200, 12)
    rc, h, _, _ = eng.key_set_new(keys3, 3)
    try:
        rc, res = eng.key_set_verify_flat(h, fl, offs, sg, None, 200)
        assert res == eng.verify_each_flat(fl, offs, sg, keys3[:32] * 200, 200)[1]
    finally:
        eng.key_set_destroy(h)


@pytest.mark.parametrize("k", [1, 3, 1024, 4096])
def test_random_indices(eng, k):
    n = 5000
    keys, fl, offs, sg, pks, idx = _signed(eng, k, n, 20 + k)
    rc, h, ok, _ = eng.key_set_new(keys, k)
    assert rc == OK and eng.key_set_len(h) == k
    try:
        for strict in (False, True):
            for device in (False, True):
                _check(eng, h, fl, offs, sg, pks, idx, n, strict=strict, device=device)
    finally:
        eng.key_set_destroy(h)


def test_many_keys_many_build_passes(eng, oracle):
    """k = 65536 keys (16 build passes of 4096) and 2^18 signatures"""
    k, n = 65536, 1 << 18
    keys, fl, offs, sg, pks, idx = _signed(eng, k, n, 31)
    rc, h, ok, weak = eng.key_set_new(keys, k)
    assert rc == OK and ok == b"\x01" * k and weak == bytes(k)
    try:
        res = _check(eng, h, fl, offs, sg, pks, idx, n)
        assert _check(eng, h, fl, offs, sg, pks, idx, n, device=True) == res
        rnd = random.Random(4)
        bad = [i for i, r in enumerate(res) if r]
        for i in bad + rnd.sample(range(n), 24):
            m = fl[int(offs[i]):int(offs[i + 1])].tobytes()
            assert oracle.verify(m, sg[64 * i:64 * i + 64].tobytes(), keys[32 * idx[i]:32 * idx[i] + 32]) == res[i]
        assert len(set(idx.tolist())) > 60000                   # the tables of every build pass are read
    finally:
        eng.key_set_destroy(h)


@pytest.fixture(scope="module")
def sized(eng):
    n = (1 << 17) + 9
    keys, fl, offs, sg, pks, idx = _signed(eng, 1024, n, 41)
    rc, h, _, _ = eng.key_set_new(keys, 1024)
    yield h, fl, offs, sg, pks, idx
    eng.key_set_destroy(h)


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, (1 << 16) - 1, 1 << 16, (1 << 16) + 1, (1 << 17) + 9])
def test_sizes(eng, sized, n):
    """the four-signatures-per-thread edges of the comb kernel and the 2^16 piece edges"""
    h, fl, offs, sg, pks, idx = sized
    o = np.ascontiguousarray(offs[:n + 1])
    s = np.ascontiguousarray(sg[:64 * n])
    p = pks[:32 * n]
    i = np.ascontiguousarray(idx[:n])
    for strict in (False, True):
        for device in (False, True):
            _check(eng, h, fl, o, s, p, i, n, strict=strict, device=device)
    rc, res = eng.key_set_verify_flat(h, fl, o, s, i, n)
    assert (rc == OK) == (not any(res))


# ---- 5. bad indices ------------------------------------------------------------------------------------------------
def test_bad_index(eng):
    import torch
    k, n = 5, 300
    keys, fl, offs, sg, pks, idx = _signed(eng, k, n, 51)
    rc, h, _, _ = eng.key_set_new(keys, k)
    lib = eng.lib
    try:
        res = (C.c_uint8 * n)()
        for pos in (0, 150, n - 1):
            bad = idx.copy(); bad[pos] = k
            before = eng.launch_count()
            assert lib.ed25519_b200_key_set_verify_flat(eng.h, h, fl.ctypes.data, offs.ctypes.data, sg.ctypes.data,
                                                        bad.ctypes.data, n, 0, res) == INVALID
            assert eng.launch_count() == before
            assert b"key index" in lib.dalek_b200_last_error(eng.h)
            ph = np.zeros(64 * n, np.uint8)
            assert lib.ed25519_b200_key_set_verify_prehashed(eng.h, h, ph.ctypes.data, None, 0, sg.ctypes.data,
                                                             bad.ctypes.data, n, 0, res) == INVALID
            assert eng.launch_count() == before
            dev = torch.device("cuda", 0)
            d = [torch.from_numpy(x).to(dev) for x in (fl, offs.view(np.int64), sg)]
            for b in (k, 0xffffffff):
                bad[pos] = b
                di = torch.from_numpy(bad.view(np.int32)).to(dev)
                assert lib.ed25519_b200_key_set_verify_flat_dev(eng.h, h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                                                di.data_ptr(), n, 0, res) == INVALID
        # the set and the context still work
        _check(eng, h, fl, offs, sg, pks, idx, n)
        _check(eng, h, fl, offs, sg, pks, idx, n, device=True)
        import curve25519_dalek_b200 as pkg
        s = pkg.VerifyingKeySet([keys[:32]], engine=eng)
        with pytest.raises(ValueError):
            s.verify_each([b"m"], [bytes(64)], indices=[1])
        s.close()
    finally:
        eng.key_set_destroy(h)


def test_argument_errors(eng):
    lib = eng.lib
    keys, fl, offs, sg, _, idx = _signed(eng, 2, 4, 61)
    h = C.c_void_p()
    assert lib.ed25519_b200_key_set_new(eng.h, keys, 0, None, None, C.byref(h)) == INVALID and not h.value
    assert lib.ed25519_b200_key_set_new(eng.h, None, 2, None, None, C.byref(h)) == INVALID and not h.value
    assert lib.ed25519_b200_key_set_new(eng.h, keys, 2, None, None, C.byref(h)) == OK and h.value
    res = (C.c_uint8 * 4)()
    try:
        assert lib.ed25519_b200_key_set_verify_flat(eng.h, h, None, None, None, None, 0, 0, None) == OK
        assert lib.ed25519_b200_key_set_verify_flat_dev(eng.h, h, None, None, None, None, 0, 0, None) == OK
        assert lib.ed25519_b200_key_set_verify_prehashed(eng.h, h, None, None, 0, None, None, 0, 0, None) == OK
        assert lib.ed25519_b200_key_set_verify_flat(eng.h, h, fl.ctypes.data, offs.ctypes.data, None, None, 4, 0, res) == INVALID
        assert lib.ed25519_b200_key_set_verify_flat(eng.h, h, fl.ctypes.data, offs.ctypes.data, sg.ctypes.data, None, 4, 0, None) == INVALID
        bad_offs = offs.copy(); bad_offs[0] = 1                                   # offsets must start at 0
        assert lib.ed25519_b200_key_set_verify_flat(eng.h, h, fl.ctypes.data, bad_offs.ctypes.data, sg.ctypes.data, None, 4, 0, res) == INVALID
        assert lib.ed25519_b200_key_set_verify_flat_dev(eng.h, h, None, None, None, None, 4, 0, res) == INVALID
        assert lib.ed25519_b200_key_set_verify_flat(eng.h, None, fl.ctypes.data, offs.ctypes.data, sg.ctypes.data, None, 4, 0, res) == INVALID
        assert lib.ed25519_b200_key_set_verify_flat(None, h, fl.ctypes.data, offs.ctypes.data, sg.ctypes.data, None, 4, 0, res) == INVALID
        ph = np.zeros(64 * 4, np.uint8)
        ctx = bytes(256)
        assert lib.ed25519_b200_key_set_verify_prehashed(eng.h, h, ph.ctypes.data, ctx, 256, sg.ctypes.data, None, 4, 0, res) == INVALID
        assert lib.ed25519_b200_key_set_verify_prehashed(eng.h, h, ph.ctypes.data, None, 3, sg.ctypes.data, None, 4, 0, res) == INVALID
    finally:
        lib.ed25519_b200_key_set_destroy(h)


# ---- 6. Ed25519ph --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("context", [None, b"", bytes(range(255))], ids=["none", "empty", "255"])
def test_prehashed(eng, context):
    k, n = 64, 700
    g = np.random.Generator(np.random.PCG64(71))
    kseeds = g.integers(0, 256, size=(k, 32), dtype=np.uint8)
    keys = eng.verifying_keys(kseeds, k)
    idx = u32(g.integers(0, k, size=n))
    phs = g.integers(0, 256, size=64 * n, dtype=np.uint8)
    rc, sigs = eng.sign_prehashed(np.ascontiguousarray(kseeds[idx]), n, phs, n, context)
    assert rc == OK
    sg = np.frombuffer(sigs, dtype=np.uint8).copy()
    for i in (0, 3, 399, n - 1):
        sg[64 * i + 9] ^= 1
    x = sg[64 * 7 + 32:64 * 8].copy(); x[31] |= 0xf0; sg[64 * 7 + 32:64 * 8] = x         # ScalarFormat
    inline = b"".join(keys[32 * t:32 * t + 32] for t in idx.tolist())
    rc, h, _, _ = eng.key_set_new(keys, k)
    try:
        for strict in (False, True):
            want = eng.verify_prehashed_each(phs, sg, inline, n, context, strict)
            assert eng.key_set_verify_prehashed(h, phs, sg, idx, n, context, strict) == want
            assert [i for i, r in enumerate(want[1]) if r] == [0, 3, 7, 399, n - 1] and want[1][7] == SCALARFMT
        # a ph signature is not a pure one over the prehash bytes, and the reverse
        msgs = [phs[64 * i:64 * i + 64].tobytes() for i in range(n)]
        fl, offs = flat(msgs)
        rc, res = eng.key_set_verify_flat(h, fl, offs, np.frombuffer(sigs, dtype=np.uint8).copy(), idx, n)
        assert rc == VERIFY and all(r == VERIFY for r in res)
        _, pure = eng.sign_batch_flat(np.ascontiguousarray(kseeds[idx]), fl, offs, n)
        assert eng.key_set_verify_flat(h, fl, offs, pure, idx, n)[1] == [OK] * n
        rc, res = eng.key_set_verify_prehashed(h, phs, pure, idx, n, context)
        assert rc == VERIFY and all(r == VERIFY for r in res)
        import curve25519_dalek_b200 as pkg
        s = pkg.VerifyingKeySet([keys[32 * t:32 * t + 32] for t in range(k)], engine=eng)
        assert s.verify_prehashed_each([phs[64 * i:64 * i + 64].tobytes() for i in range(n)],
                                       [sigs[64 * i:64 * i + 64] for i in range(n)], idx.tolist(), context) == [OK] * n
        assert s.verify_prehashed_each(phs[64:128].tobytes(), sigs[64:128], int(idx[1]), context, strict=True) == OK
        with pytest.raises(ValueError):
            s.verify_prehashed_each([phs[:64].tobytes()], [sigs[:64]], [0], bytes(256))
        s.close()
    finally:
        eng.key_set_destroy(h)


# ---- 7. options ----------------------------------------------------------------------------------------------------
def test_options_do_not_change_results(eng, vectors, oracle):
    msgs, sigs, keys = vectors
    decodable = [kk for kk in dict.fromkeys(keys) if oracle.decompress(kk) is not None]
    pos = {kk: i for i, kk in enumerate(decodable)}
    use = [i for i, kk in enumerate(keys) if kk in pos]
    m, s, idx = [msgs[i] for i in use], [sigs[i] for i in use], [pos[keys[i]] for i in use]
    ks = KeySet(eng, decodable)
    try:
        base = {st: ks.verify(m, s, idx, st) for st in (False, True)}
        for opt, vals in (("each_comb", (0, 1, 2)), ("field_f64", (0, 1))):
            for v in vals:
                eng.set_option(opt, v)
                try:
                    for st in (False, True):
                        assert ks.verify(m, s, idx, st) == base[st], (opt, v, st)
                        assert ks.verify(m, s, idx, st, device=True) == base[st], (opt, v, st)
                finally:
                    eng.set_option(opt, 1)
    finally:
        ks.close()


# ---- 8. lifecycle --------------------------------------------------------------------------------------------------
def test_destroy_after_engine_close_and_foreign_context(eng):
    import curve25519_dalek_b200 as pkg
    keys, fl, offs, sg, pks, idx = _signed(eng, 4, 50, 81)
    e2 = pkg.Engine(0)
    rc, h2, _, _ = e2.key_set_new(keys, 4)
    assert rc == OK
    res = (C.c_uint8 * 50)()
    assert eng.lib.ed25519_b200_key_set_verify_flat(eng.h, h2, fl.ctypes.data, offs.ctypes.data, sg.ctypes.data,
                                                    idx.ctypes.data, 50, 0, res) == INVALID
    assert b"context" in eng.lib.dalek_b200_last_error(eng.h)
    ph = np.zeros(64 * 50, np.uint8)
    assert eng.lib.ed25519_b200_key_set_verify_prehashed(eng.h, h2, ph.ctypes.data, None, 0, sg.ctypes.data, idx.ctypes.data,
                                                         50, 0, res) == INVALID
    assert eng.lib.ed25519_b200_key_set_verify_flat_dev(eng.h, h2, None, None, None, None, 0, 0, None) == INVALID
    _check(e2, h2, fl, offs, sg, pks, idx, 50)
    s2 = pkg.VerifyingKeySet([keys[:32]], engine=e2)
    e2.close()
    e2.key_set_destroy(h2)                                       # after the context: must not touch it
    s2.close()
    eng.lib.ed25519_b200_key_set_destroy(None)
    assert eng.lib.ed25519_b200_key_set_len(None) == 0
    rc, h, _, _ = eng.key_set_new(keys, 4)                       # this engine is unaffected
    _check(eng, h, fl, offs, sg, pks, idx, 50)
    eng.key_set_destroy(h)


def test_two_contexts_on_two_threads(eng):
    import curve25519_dalek_b200 as pkg
    errs = []

    def work(seed):
        try:
            e = pkg.Engine(0)
            keys, fl, offs, sg, pks, idx = _signed(e, 97, 20000, seed)
            rc, h, _, _ = e.key_set_new(keys, 97)
            for _ in range(5):
                _check(e, h, fl, offs, sg, pks, idx, 20000)
            e.key_set_destroy(h)
            e.close()
        except Exception as exc:                                 # reported below
            errs.append(repr(exc))

    ts = [threading.Thread(target=work, args=(s,)) for s in (91, 92)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_reuse_over_many_calls(eng):
    keys, fl, offs, sg, pks, idx = _signed(eng, 300, 70000, 101)
    rc, h, _, _ = eng.key_set_new(keys, 300)
    rnd = random.Random(7)
    try:
        for c in range(50):
            n = rnd.choice([0, 1, 7, 128, 1000, 4097, 66000]) if c % 10 else 70000
            lo = rnd.randrange(0, 70000 - n + 1)
            o = np.ascontiguousarray(offs[lo:lo + n + 1] - offs[lo])
            f = np.ascontiguousarray(fl[int(offs[lo]):int(offs[lo + n]) + 1])
            _check(eng, h, f, o, np.ascontiguousarray(sg[64 * lo:64 * (lo + n)]), pks[32 * lo:32 * (lo + n)],
                   np.ascontiguousarray(idx[lo:lo + n]), n, strict=bool(c & 1), device=(c % 3 == 0))
    finally:
        eng.key_set_destroy(h)


# ---- 9. round trip with the GPU signer -----------------------------------------------------------------------------
def test_round_trip_with_gpu_signer(eng):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(9)
    seeds = [rnd.randbytes(32) for _ in range(1024)]
    keys = pkg.ed25519_verifying_keys(seeds, engine=eng)
    per = 3
    msgs = [b"vote %d round %d" % (i, j) + rnd.randbytes(j * 17) for i in range(1024) for j in range(per)]
    sigs = pkg.ed25519_sign([seeds[i // per] for i in range(len(msgs))], msgs, engine=eng)
    idx = [i // per for i in range(len(msgs))]
    s = pkg.VerifyingKeySet(keys, engine=eng)
    try:
        assert len(s) == 1024 and not any(s.is_weak(i) for i in range(1024))
        assert s.verify_each(msgs, sigs, idx) == [OK] * len(msgs)
        assert s.verify_each(msgs, sigs, idx, strict=True) == [OK] * len(msgs)
        assert s.verify_each(msgs[5], sigs[5], idx[5]) == OK
        assert s.verify_each(msgs[5], sigs[5], idx[5] + 1) == VERIFY
        bad = list(msgs); bad[1234] = bad[1234] + b"!"
        res = s.verify_each(bad, sigs, idx)
        assert [i for i, r in enumerate(res) if r] == [1234]
        assert s.verify_each([msgs[0], msgs[1]], [sigs[0], sigs[1]]) == [OK, OK]     # indices None: key 0
        assert s.verify_each([], []) == []
    finally:
        s.close()
