"""GPU signing-key sets and hazmat signing: ed25519_b200_signing_key_set_* against ed25519_b200_sign_flat, the C oracle and
the Ed25519ph oracle; ed25519_b200_expanded_verifying_keys / raw_sign_flat / raw_sign_prehashed against the raw_sign model
(tests/raw_sign_model.py) on arbitrary ExpandedSecretKey bytes; keypair validation, bad indices and the set's lifecycle."""
import ctypes as C
import hashlib
import random
import threading

import numpy as np
import pytest

import ed25519ph_oracle
import oracle_lib
from raw_sign_model import RawSignModel, clamp

pytestmark = pytest.mark.gpu

OK, POINTDEC, CTXLEN, MISMATCH, INVALID = 0, 4, 5, 6, -1
SEED, KEYPAIR, EXPANDED = 0, 1, 2
L = 2**252 + 27742317777372353535851937790883648493


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
def model(orc):
    return RawSignModel(orc)


def flat(msgs):
    offs = np.zeros(len(msgs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m) for m in msgs]) if msgs else []
    return np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy(), offs


def split(raw, k):
    return [raw[k * i:k * i + k] for i in range(len(raw) // k)]


def new_set(eng, keys, form):
    rc, h, status = eng.signing_key_set_new(b"".join(keys), len(keys), form)
    assert rc == OK and h is not None and status == bytes(len(keys))
    return h


def set_sign(eng, h, msgs, idx):
    fl, offs = flat(msgs)
    ib = np.asarray(idx, dtype=np.uint32) if idx is not None else None
    return split(eng.signing_key_set_sign_flat(h, fl, offs, ib, len(msgs)), 64)


def per_message_sign(eng, seeds, msgs, idx):
    fl, offs = flat(msgs)
    return split(eng.sign_flat(b"".join(seeds[i] for i in idx), len(msgs), fl, offs, len(msgs)), 64)


# ---- 1. seeds: the same bytes as sign_flat with each message's seed, and as the oracle ---------------------------------
@pytest.mark.parametrize("k,n", [(1, 3000), (2, 3000), (1000, 20000), (70000, (1 << 17) + 3)])
def test_set_from_seeds_matches_sign_flat_and_oracle(eng, orc, k, n):
    rnd = random.Random(k)
    seeds = [rnd.randbytes(32) for _ in range(k)]
    msgs = [rnd.randbytes(rnd.randrange(0, 90)) for _ in range(n)]
    idx = [rnd.randrange(k) for _ in range(n)]
    h = new_set(eng, seeds, SEED)
    try:
        sigs = set_sign(eng, h, msgs, idx)
        assert sigs == per_message_sign(eng, seeds, msgs, idx)
        for i in sorted(rnd.sample(range(n), min(n, 400))):
            assert sigs[i] == orc.sign(msgs[i], seeds[idx[i]]), i
        pks = split(eng.signing_key_set_verifying_keys(h), 32)
        assert pks == split(eng.verifying_keys(b"".join(seeds), k), 32)
        fl, offs = flat(msgs)
        rc, res = eng.verify_each_flat(fl, offs, b"".join(sigs), b"".join(pks[i] for i in idx), n, strict=True)
        assert rc == OK and not any(res)
    finally:
        eng.signing_key_set_destroy(h)


def test_message_lengths_at_block_boundaries(eng, orc):
    rnd = random.Random(5)
    lens = [0, 47, 48, 79, 80, 175, 176, 207, 208, 111, 112, 239, 240, 1 << 20, 3, 128, 255, 256]
    msgs = [rnd.randbytes(k) for k in lens]
    seeds = [rnd.randbytes(32) for _ in range(3)]
    idx = [i % 3 for i in range(len(msgs))]
    h = new_set(eng, seeds, SEED)
    sigs = set_sign(eng, h, msgs, idx)
    eng.signing_key_set_destroy(h)
    for i, m in enumerate(msgs):
        assert sigs[i] == orc.sign(m, seeds[idx[i]]), lens[i]


def test_null_indices_mean_key_zero(eng, orc):
    rnd = random.Random(6)
    seeds = [rnd.randbytes(32) for _ in range(5)]
    msgs = [rnd.randbytes(rnd.randrange(100)) for _ in range(300)]
    h = new_set(eng, seeds, SEED)
    sigs = set_sign(eng, h, msgs, None)
    eng.signing_key_set_destroy(h)
    assert sigs == per_message_sign(eng, seeds, msgs, [0] * len(msgs))
    assert sigs[7] == orc.sign(msgs[7], seeds[0])


# ---- 2. Ed25519ph ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("clen", [0, 1, 255])
def test_prehashed_contexts(eng, pho, clen):
    rnd = random.Random(10 + clen)
    seeds = [rnd.randbytes(32) for _ in range(7)]
    ctx = rnd.randbytes(clen)
    phs = [rnd.randbytes(64) for _ in range(500)]
    idx = np.array([rnd.randrange(7) for _ in phs], dtype=np.uint32)
    h = new_set(eng, seeds, SEED)
    rc, raw = eng.signing_key_set_sign_prehashed(h, b"".join(phs), idx, len(phs), ctx)
    assert rc == OK
    for i, sig in enumerate(split(raw, 64)):
        assert (0, sig) == pho.sign_prehashed(seeds[idx[i]], phs[i], ctx), i
    out = (C.c_uint8 * 64).from_buffer_copy(b"\xaa" * 64)
    assert eng.lib.ed25519_b200_signing_key_set_sign_prehashed(eng.h, h, phs[0], bytes(256), 256, None, 1, out) == CTXLEN
    assert bytes(out) == b"\xaa" * 64                              # nothing written
    eng.signing_key_set_destroy(h)


# ---- 3. expanded keys and the hazmat calls ----------------------------------------------------------------------------
def test_from_expanded_of_seed_hash_equals_from_seeds(eng):
    rnd = random.Random(20)
    seeds = [rnd.randbytes(32) for _ in range(50)]
    msgs = [rnd.randbytes(rnd.randrange(200)) for _ in range(1000)]
    idx = [rnd.randrange(50) for _ in msgs]
    h1 = new_set(eng, seeds, SEED)
    h2 = new_set(eng, [hashlib.sha512(s).digest() for s in seeds], EXPANDED)
    assert eng.signing_key_set_verifying_keys(h1) == eng.signing_key_set_verifying_keys(h2)
    assert set_sign(eng, h1, msgs, idx) == set_sign(eng, h2, msgs, idx)
    eng.signing_key_set_destroy(h1)
    eng.signing_key_set_destroy(h2)


def _edge_esks(rnd):
    """Arbitrary 64-byte ExpandedSecretKeys: random halves (clamp bits set wrongly), all-zero and all-0xff halves, and low
    halves whose clamped value is a multiple of l plus small values (every clamped value is >= 2^254 > l)."""
    out = [rnd.randbytes(64) for _ in range(40)]
    out += [bytes(64), b"\xff" * 64, bytes(32) + b"\xff" * 32, b"\xff" * 32 + bytes(32)]
    for j in (0, 1, 2):
        x = 4 * L + 4 + 8 * j                                        # clamp(x) = x: bits 0-2 and 255 clear, bit 254 set
        assert int.from_bytes(clamp(x.to_bytes(32, "little")), "little") == x
        out.append(x.to_bytes(32, "little") + rnd.randbytes(32))
    lo = bytearray(rnd.randbytes(32)); lo[0] |= 7; lo[31] |= 0x80; lo[31] &= ~0x40 & 0xff   # every clamp bit wrong
    out.append(bytes(lo) + rnd.randbytes(32))
    return out


def test_raw_sign_matches_the_model(eng, model):
    rnd = random.Random(21)
    esks = _edge_esks(rnd)
    n = len(esks)
    vks = split(eng.expanded_verifying_keys(b"".join(esks), n), 32)
    assert vks == [model.verifying_key(e) for e in esks]
    msgs = [rnd.randbytes(rnd.randrange(300)) for _ in range(n)]
    fl, offs = flat(msgs)
    sigs = split(eng.raw_sign_flat(b"".join(esks), b"".join(vks), n, fl, offs, n), 64)
    assert sigs == [model.raw_sign(e, m, v) for e, m, v in zip(esks, msgs, vks)]
    one = split(eng.raw_sign_flat(esks[1], vks[1], 1, fl, offs, n), 64)          # one key for every message
    assert one == [model.raw_sign(esks[1], m, vks[1]) for m in msgs]
    phs = [rnd.randbytes(64) for _ in range(n)]
    rc, raw = eng.raw_sign_prehashed(b"".join(esks), b"".join(vks), n, b"".join(phs), n, b"ctx")
    assert rc == OK and split(raw, 64) == [model.raw_sign_prehashed(e, p, v, b"ctx") for e, p, v in zip(esks, phs, vks)]
    assert eng.raw_sign_prehashed(esks[0], vks[0], 1, phs[0], 1, bytes(256))[0] == CTXLEN
    h = new_set(eng, esks, EXPANDED)                               # the set: the same bytes under the derived keys
    assert split(eng.signing_key_set_verifying_keys(h), 32) == vks
    idx = [rnd.randrange(n) for _ in msgs]
    assert set_sign(eng, h, msgs, idx) == [model.raw_sign(esks[i], m, vks[i]) for i, m in zip(idx, msgs)]
    eng.signing_key_set_destroy(h)


def test_raw_sign_with_a_mismatched_key_gives_the_reference_bytes(eng, orc, model):
    rnd = random.Random(22)
    esks = [rnd.randbytes(64) for _ in range(64)]
    other = [orc.public_key(rnd.randbytes(32)) for _ in esks]     # valid keys of other secrets
    msgs = [rnd.randbytes(rnd.randrange(150)) for _ in esks]
    fl, offs = flat(msgs)
    sigs = split(eng.raw_sign_flat(b"".join(esks), b"".join(other), 64, fl, offs, 64), 64)
    assert sigs == [model.raw_sign(e, m, v) for e, m, v in zip(esks, msgs, other)]


def test_raw_sign_across_pieces(eng, model):
    rnd = random.Random(23)
    n = (1 << 17) + 3
    gen = np.random.Generator(np.random.PCG64(23))
    esks = gen.integers(0, 256, size=(n, 64), dtype=np.uint8)
    vks = np.frombuffer(eng.expanded_verifying_keys(esks, n), dtype=np.uint8).reshape(n, 32)
    msgs = [rnd.randbytes(rnd.randrange(64)) for _ in range(n)]
    fl, offs = flat(msgs)
    sigs = split(eng.raw_sign_flat(esks, vks, n, fl, offs, n), 64)
    for i in sorted(rnd.sample(range(n), 300)) + [65535, 65536, n - 1]:
        e = esks[i].tobytes()
        assert vks[i].tobytes() == model.verifying_key(e)
        assert sigs[i] == model.raw_sign(e, msgs[i], vks[i].tobytes()), i


# ---- 4. keypairs -------------------------------------------------------------------------------------------------------
def test_keypair_status(eng, orc):
    rnd = random.Random(30)
    seeds = [rnd.randbytes(32) for _ in range(8)]
    pks = [orc.public_key(s) for s in seeds]
    good = [s + p for s, p in zip(seeds, pks)]
    h = new_set(eng, good, KEYPAIR)
    msgs = [b"abc", b""]
    assert set_sign(eng, h, msgs, [3, 5]) == [orc.sign(b"abc", seeds[3]), orc.sign(b"", seeds[5])]
    assert split(eng.signing_key_set_verifying_keys(h), 32) == pks
    eng.signing_key_set_destroy(h)
    undecodable = (2).to_bytes(32, "little")                        # y = 2 is not on the curve
    negated = bytearray(pks[2]); negated[31] ^= 0x80                 # -A: decodes, another point
    # y = p + 1, a non-canonical encoding of the identity: it decodes, and equality is on bytes.  (A seed's own key has a
    # y far above 18, so it has no non-canonical encoding to test with; any encoding other than the derived bytes is a
    # mismatch once it decodes.)
    noncanonical = (2**255 - 19 + 1).to_bytes(32, "little")
    cases = [(seeds[0] + pks[1], MISMATCH), (seeds[1] + undecodable, POINTDEC), (seeds[2] + bytes(negated), MISMATCH),
             (seeds[3] + noncanonical, MISMATCH)]
    for kp, want in cases:
        rc, hh, status = eng.signing_key_set_new(kp, 1, KEYPAIR)
        assert (rc, hh, status) == (want, None, bytes([want]))
    mix = [good[0], cases[2][0], good[1], cases[1][0], cases[0][0]]
    rc, hh, status = eng.signing_key_set_new(b"".join(mix), 5, KEYPAIR)
    assert (rc, hh, list(status)) == (MISMATCH, None, [0, MISMATCH, 0, POINTDEC, MISMATCH])
    import curve25519_dalek_b200 as pkg
    with pytest.raises(pkg.SignatureError) as e:
        pkg.SigningKeySet.from_keypair_bytes(mix[2:], engine=eng)
    assert e.value.code == POINTDEC and e.value.kind == "PointDecompression" and "key 1" in str(e.value)
    with pytest.raises(pkg.SignatureError) as e:
        pkg.SigningKeySet.from_keypair_bytes(mix, engine=eng)
    assert e.value.kind == "MismatchedKeypair" and "key 1" in str(e.value)


# ---- 5. indices and arguments ------------------------------------------------------------------------------------------
def test_bad_indices(eng, orc):
    import torch
    rnd = random.Random(40)
    seeds = [rnd.randbytes(32) for _ in range(4)]
    msgs = [rnd.randbytes(rnd.randrange(80)) for _ in range(1000)]
    fl, offs = flat(msgs)
    h = new_set(eng, seeds, SEED)
    idx = np.array([rnd.randrange(4) for _ in msgs], dtype=np.uint32)
    idx[17] = 4
    out = (C.c_uint8 * (64 * 1000)).from_buffer_copy(b"\xaa" * 64000)
    lib = eng.lib
    assert lib.ed25519_b200_signing_key_set_sign_flat(eng.h, h, fl.ctypes.data, offs.ctypes.data, idx.ctypes.data, 1000, out) == INVALID
    assert bytes(out) == b"\xaa" * 64000                           # refused before any work
    assert lib.ed25519_b200_signing_key_set_sign_prehashed(eng.h, h, bytes(64 * 1000), None, 0, idx.ctypes.data, 1000, out) == INVALID
    dev = torch.device("cuda", 0)
    d_fl, d_offs = torch.from_numpy(fl).to(dev), torch.from_numpy(offs.view(np.int64)).to(dev)
    d_out = torch.full((64 * 1000,), 0xaa, dtype=torch.uint8, device=dev)
    for bad in (4, 0xffffffff):
        idx[17] = bad
        d_idx = torch.from_numpy(idx.view(np.int32)).to(dev)
        with pytest.raises(Exception):
            eng.signing_key_set_sign_flat(h, d_fl.data_ptr(), d_offs.data_ptr(), d_idx.data_ptr(), 1000, device_ptrs=True,
                                          out=d_out.data_ptr())
        got = split(d_out.cpu().numpy().tobytes(), 64)
        assert got[17] == bytes(64)                                # zero bytes, never a signature under another key
        good = [i for i in range(1000) if i != 17]
        want = per_message_sign(eng, seeds, [msgs[i] for i in good], [int(idx[i]) for i in good])
        assert [got[i] for i in good] == want
    idx[17] = 3
    d_idx = torch.from_numpy(idx.view(np.int32)).to(dev)
    assert eng.signing_key_set_sign_flat(h, d_fl.data_ptr(), d_offs.data_ptr(), d_idx.data_ptr(), 1000, device_ptrs=True,
                                         out=d_out.data_ptr()) is None
    assert split(d_out.cpu().numpy().tobytes(), 64) == set_sign(eng, h, msgs, idx)
    eng.signing_key_set_destroy(h)


def test_device_call_matches_host_call(eng):
    import torch
    rnd = random.Random(41)
    k, n = 300, (1 << 17) + 3
    seeds = [rnd.randbytes(32) for _ in range(k)]
    msgs = [rnd.randbytes(rnd.randrange(40)) for _ in range(n)]
    idx = np.array([rnd.randrange(k) for _ in range(n)], dtype=np.uint32)
    fl, offs = flat(msgs)
    h = new_set(eng, seeds, SEED)
    dev = torch.device("cuda", 0)
    d = [torch.from_numpy(x).to(dev) for x in (fl, offs.view(np.int64), idx.view(np.int32))]
    d_out = torch.empty(64 * n, dtype=torch.uint8, device=dev)
    eng.signing_key_set_sign_flat(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), n, device_ptrs=True, out=d_out.data_ptr())
    assert d_out.cpu().numpy().tobytes() == eng.signing_key_set_sign_flat(h, fl, offs, idx, n)
    eng.signing_key_set_sign_flat(h, d[0].data_ptr(), d[1].data_ptr(), None, n, device_ptrs=True, out=d_out.data_ptr())
    assert d_out.cpu().numpy().tobytes() == eng.signing_key_set_sign_flat(h, fl, offs, None, n)
    eng.signing_key_set_destroy(h)


def test_argument_checks(eng):
    lib, hc = eng.lib, eng.h
    out = C.c_void_p()
    seeds = bytes(64)
    new = lib.ed25519_b200_signing_key_set_new
    assert new(hc, seeds, 0, SEED, None, C.byref(out)) == INVALID and not out.value          # k = 0
    assert new(hc, seeds, 2, 3, None, C.byref(out)) == INVALID and not out.value             # unknown form
    assert new(hc, seeds, 2, -1, None, C.byref(out)) == INVALID
    assert new(hc, None, 2, SEED, None, C.byref(out)) == INVALID
    assert new(hc, seeds, 2, SEED, None, None) == INVALID
    assert new(hc, seeds, 2, SEED, None, C.byref(out)) == OK and out.value                  # status may be NULL
    h = out
    assert lib.ed25519_b200_signing_key_set_len(h) == 2 and lib.ed25519_b200_signing_key_set_len(None) == 0
    assert lib.ed25519_b200_signing_key_set_verifying_keys(h, None) == INVALID
    assert lib.ed25519_b200_signing_key_set_verifying_keys(None, (C.c_uint8 * 64)()) == INVALID
    sf = lib.ed25519_b200_signing_key_set_sign_flat
    fl, offs = np.zeros(8, np.uint8), np.array([0, 1, 2], dtype=np.uint64)
    res = (C.c_uint8 * 128)()
    assert sf(hc, h, fl.ctypes.data, offs.ctypes.data, None, 2, res) == OK
    assert sf(hc, h, fl.ctypes.data, offs.ctypes.data, None, 2, None) == INVALID
    assert sf(hc, h, None, offs.ctypes.data, None, 2, res) == INVALID
    assert sf(hc, None, fl.ctypes.data, offs.ctypes.data, None, 2, res) == INVALID
    assert sf(hc, h, None, None, None, 0, None) == OK                                        # n = 0
    sp = lib.ed25519_b200_signing_key_set_sign_prehashed
    assert sp(hc, h, bytes(128), None, 1, None, 2, res) == INVALID                          # NULL context, non-zero length
    assert sp(hc, h, bytes(128), None, 0, None, 2, res) == OK
    rf = lib.ed25519_b200_raw_sign_flat
    assert rf(hc, bytes(192), bytes(96), 3, fl.ctypes.data, offs.ctypes.data, 2, res) == INVALID   # n_keys not in {1, n}
    assert rf(hc, bytes(128), None, 2, fl.ctypes.data, offs.ctypes.data, 2, res) == INVALID
    assert rf(hc, bytes(128), bytes(64), 2, fl.ctypes.data, offs.ctypes.data, 2, res) == OK
    assert rf(hc, None, None, 0, None, None, 0, None) == OK
    rp = lib.ed25519_b200_raw_sign_prehashed
    assert rp(hc, bytes(64), bytes(32), 1, bytes(128), 2, None, 0, res) == OK
    assert rp(hc, bytes(64), None, 1, bytes(128), 2, None, 0, res) == INVALID
    assert lib.ed25519_b200_expanded_verifying_keys(hc, None, 1, res) == INVALID
    assert lib.ed25519_b200_expanded_verifying_keys(hc, None, 0, None) == OK
    lib.ed25519_b200_signing_key_set_destroy(h)
    lib.ed25519_b200_signing_key_set_destroy(None)


# ---- 6. lifecycle ------------------------------------------------------------------------------------------------------
def test_foreign_context_and_destroy_after_engine_close(eng, orc):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(50)
    seeds = [rnd.randbytes(32) for _ in range(3)]
    e2 = pkg.Engine(0)
    h2 = new_set(e2, seeds, SEED)
    fl, offs = flat([b"m"])
    res = (C.c_uint8 * 64)()
    assert eng.lib.ed25519_b200_signing_key_set_sign_flat(eng.h, h2, fl.ctypes.data, offs.ctypes.data, None, 1, res) == INVALID
    assert b"context" in eng.lib.dalek_b200_last_error(eng.h)
    assert eng.lib.ed25519_b200_signing_key_set_sign_prehashed(eng.h, h2, bytes(64), None, 0, None, 1, res) == INVALID
    assert eng.lib.ed25519_b200_signing_key_set_sign_flat_dev(eng.h, h2, None, None, None, 0, None) == INVALID
    assert set_sign(e2, h2, [b"m"], [2]) == [orc.sign(b"m", seeds[2])]
    s2 = pkg.SigningKeySet.from_seeds(seeds, engine=e2)
    e2.close()
    e2.signing_key_set_destroy(h2)                                 # after the context: must not touch it
    s2.close()
    s = pkg.SigningKeySet.from_seeds(seeds, engine=eng)           # this engine is unaffected
    assert s.sign(b"m", 1) == orc.sign(b"m", seeds[1])
    s.close()


def test_reuse_over_many_calls(eng, orc):
    rnd = random.Random(51)
    seeds = [rnd.randbytes(32) for _ in range(100)]
    msgs = [rnd.randbytes(rnd.randrange(64)) for _ in range(5000)]
    idx = [rnd.randrange(100) for _ in msgs]
    h = new_set(eng, seeds, SEED)
    first = set_sign(eng, h, msgs, idx)
    for _ in range(10):
        fl, offs = flat([b"other"] * 77)                           # other calls in between use the same workspaces
        eng.sign_flat(rnd.randbytes(32), 1, fl, offs, 77)
        assert set_sign(eng, h, msgs, idx) == first
    assert first[9] == orc.sign(msgs[9], seeds[idx[9]])
    eng.signing_key_set_destroy(h)


def test_two_contexts_on_two_threads(eng, orc):
    import curve25519_dalek_b200 as pkg
    errs = []

    def work(seed):
        try:
            rnd = random.Random(seed)
            e = pkg.Engine(0)
            seeds = [rnd.randbytes(32) for _ in range(50)]
            msgs = [rnd.randbytes(rnd.randrange(64)) for _ in range(20000)]
            idx = [rnd.randrange(50) for _ in msgs]
            h = new_set(e, seeds, SEED)
            want = per_message_sign(e, seeds, msgs, idx)
            for _ in range(5):
                assert set_sign(e, h, msgs, idx) == want
            e.signing_key_set_destroy(h)
            e.close()
        except Exception as exc:                                   # reported below
            errs.append(repr(exc))

    ts = [threading.Thread(target=work, args=(s,)) for s in (91, 92)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


# ---- 7. the Python layer -----------------------------------------------------------------------------------------------
def test_python_functions(eng, orc, pho, model):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(60)
    seeds = [rnd.randbytes(32) for _ in range(3)]
    msgs = [b"", b"abc", rnd.randbytes(500)]
    s = pkg.SigningKeySet.from_seeds(seeds, engine=eng)
    assert len(s) == 3
    assert s.verifying_keys() == [orc.public_key(x) for x in seeds]
    assert s.verifying_key(2) == orc.public_key(seeds[2])
    with pytest.raises(IndexError):
        s.verifying_key(3)
    assert s.sign(b"abc") == orc.sign(b"abc", seeds[0])
    assert s.sign(b"abc", 2) == orc.sign(b"abc", seeds[2])
    assert s.sign(msgs, [2, 0, 1]) == [orc.sign(m, seeds[i]) for m, i in zip(msgs, [2, 0, 1])]
    assert s.sign([]) == []
    with pytest.raises(ValueError):
        s.sign(msgs, [0, 3, 1])
    with pytest.raises(ValueError):
        s.sign(msgs, [0, 1])
    hs = [hashlib.sha512(m) for m in msgs]
    assert s.sign_prehashed(hs[1], 1, b"ctx") == pho.sign_prehashed(seeds[1], hs[1].digest(), b"ctx")[1]
    assert s.sign_prehashed(hs, [0, 1, 2]) == [pho.sign_prehashed(x, h.digest(), b"")[1] for x, h in zip(seeds, hs)]
    with pytest.raises(pkg.SignatureError) as e:
        s.sign_prehashed(hs[0], 0, bytes(256))
    assert e.value.code == CTXLEN
    s.close()
    s.close()
    esks = [rnd.randbytes(64) for _ in range(3)]
    vks = pkg.ed25519_expanded_verifying_keys(esks, engine=eng)
    assert vks == [model.verifying_key(e) for e in esks]
    assert pkg.ed25519_expanded_verifying_keys(esks[0], engine=eng) == vks[0]
    assert pkg.ed25519_raw_sign(esks[0], b"abc", vks[0], engine=eng) == model.raw_sign(esks[0], b"abc", vks[0])
    assert pkg.ed25519_raw_sign(esks, msgs, vks, engine=eng) == [model.raw_sign(e, m, v) for e, m, v in zip(esks, msgs, vks)]
    assert pkg.ed25519_raw_sign(esks[1], msgs, vks[1], engine=eng) == [model.raw_sign(esks[1], m, vks[1]) for m in msgs]
    assert pkg.ed25519_raw_sign_prehashed(esks, hs, vks, b"c", engine=eng) == \
        [model.raw_sign_prehashed(e, h.digest(), v, b"c") for e, h, v in zip(esks, hs, vks)]
    with pytest.raises(pkg.SignatureError):
        pkg.ed25519_raw_sign_prehashed(esks[0], hs[0], vks[0], bytes(256), engine=eng)
    with pytest.raises(ValueError):
        pkg.ed25519_raw_sign(esks[:2], msgs, vks[:2], engine=eng)
    x = pkg.SigningKeySet.from_expanded(esks, engine=eng)
    assert x.verifying_keys() == vks and x.sign(b"q", 1) == model.raw_sign(esks[1], b"q", vks[1])
    x.close()
    kp = pkg.SigningKeySet.from_keypair_bytes([sd + orc.public_key(sd) for sd in seeds], engine=eng)
    assert kp.sign(msgs, [1, 1, 1]) == [orc.sign(m, seeds[1]) for m in msgs]
    kp.close()
    with pytest.raises(ValueError):
        pkg.SigningKeySet.from_seeds([], engine=eng)
