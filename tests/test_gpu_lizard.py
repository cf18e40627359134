"""Lizard and the Elligator inverse on the GPU: every golden vector through the C ABI and the Python methods, map_to_curve
against the hash-to-group fixtures, oracle parity on batches of several pieces (RISTRETTO and EXTENDED input with random
representatives and Z), the round trip on 2^20 payloads, the inverse's properties, coset and scaling invariance of decode,
undecodable encodings at piece slots, an ElGamal-style chain through mul_batch, and argument checks."""
import ctypes as C
import json
import os
import random

import pytest

import h2c_model as H
import lizard_oracle
import lizard_model as L

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GROUP_L = 2**252 + 27742317777372353535851937790883648493
FMT = {"extended": 1, "ristretto": 2}
PIECE = 2**16


@pytest.fixture(scope="module")
def pkg():
    import curve25519_dalek_b200 as pkg
    return pkg


@pytest.fixture(scope="module")
def eng(pkg):
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "lizard.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def ho():
    return lizard_oracle.load()


def split(raw, w):
    return [raw[i:i + w] for i in range(0, len(raw), w)]


def test_golden_vectors_c_abi_and_python(eng, pkg, golden):
    kats = golden["lizard_encode_kat"]
    datas = [bytes.fromhex(k["data"]) for k in kats]
    assert [x.hex() for x in split(eng.ristretto_lizard_encode_batch(b"".join(datas), len(datas)), 32)] == [k["out"] for k in kats]
    assert [x.hex() for x in pkg.RistrettoPoint.lizard_encode_batch(datas, engine=eng)] == [k["out"] for k in kats]
    assert pkg.RistrettoPoint.lizard_decode_batch([bytes.fromhex(k["out"]) for k in kats], engine=eng) == datas
    ins = [bytes.fromhex(v["in"]) for v in golden["map_to_curve"]]
    want = [v["out"] for v in golden["map_to_curve"]]
    assert [x.hex() for x in split(eng.ristretto_map_to_curve_batch(b"".join(ins), len(ins)), 32)] == want
    assert [x.hex() for x in pkg.RistrettoPoint.map_to_curve_batch(ins, engine=eng)] == want
    for fmt in ("ristretto", "extended"):
        vs = [v for v in golden["points"] if v["fmt"] == fmt]
        pts = b"".join(bytes.fromhex(v["point"]) for v in vs)
        rc, raw, st = eng.ristretto_lizard_decode_batch(pts, len(vs), FMT[fmt])
        assert rc == 1                                   # every set holds a None
        assert list(st) == [v["status"] for v in vs]
        assert [x.hex() for x in split(raw, 16)] == [v["decode"] or "00" * 16 for v in vs]
        rc, raw, masks = eng.ristretto_map_to_curve_inverse_batch(pts, len(vs), FMT[fmt])
        assert rc == (1 if any(v["status"] == 2 for v in vs) else 0)
        assert masks == [v["mask"] for v in vs]
        for i, v in enumerate(vs):
            assert [c.hex() for c in split(raw[512 * i:512 * i + 512], 32)] == [x or "00" * 32 for x in v["inverse"]], v["label"]
    # the Python methods on the decodable CompressedRistretto vectors
    vs = [v for v in golden["points"] if v["fmt"] == "ristretto" and v["status"] != 2]
    encs = [bytes.fromhex(v["point"]) for v in vs]
    assert pkg.RistrettoPoint.lizard_decode_batch(encs, engine=eng) == [None if v["decode"] is None else bytes.fromhex(v["decode"])
                                                                         for v in vs]
    got = pkg.RistrettoPoint.map_to_curve_inverse_batch(encs, engine=eng)
    assert got == [[None if x is None else bytes.fromhex(x) for x in v["inverse"]] for v in vs]
    bad = [bytes.fromhex(v["point"]) for v in golden["points"] if v["status"] == 2]
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.lizard_decode_batch(bad[:1], engine=eng)
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.map_to_curve_inverse_batch(bad[:1], engine=eng)


def test_map_to_curve_against_hash_to_group_fixtures(eng):
    with open(os.path.join(ROOT, "tests", "golden", "hash_to_curve.json")) as f:
        h2c = json.load(f)
    ins = [bytes.fromhex(v["r0"]) for v in h2c["ristretto_elligator_sage"]] + [bytes.fromhex(h) for h in h2c["d_zero_halves"]]
    want = [v["out"] for v in h2c["ristretto_elligator_sage"]] + [H.ristretto_elligator(bytes.fromhex(h)).hex() for h in h2c["d_zero_halves"]]
    assert len(ins) == 20
    assert [x.hex() for x in split(eng.ristretto_map_to_curve_batch(b"".join(ins), len(ins)), 32)] == want


def _random_points(rnd, ho, n_pool):
    """A pool of points, half of them Lizard encodings: (CompressedRistretto, extended limbs of a random representative)."""
    datas = [rnd.randbytes(16) for _ in range(n_pool // 2)]
    encs = ho.lizard_encode_batch(datas) + [H.from_uniform_bytes(rnd.randbytes(64)) for _ in range(n_pool - n_pool // 2)]
    ext = [L.limbs_bytes(L.scale(L.coset4(L.ristretto_decode(e))[rnd.randrange(4)], rnd.randrange(1, L.p))) for e in encs]
    return encs, ext


def test_oracle_parity_across_pieces(eng, ho):
    rnd = random.Random(21)
    n = 2 * PIECE + 4099                                   # three pieces
    # map_to_curve and encode
    pool32 = [rnd.randbytes(32) for _ in range(4096)]
    pool16 = [rnd.randbytes(16) for _ in range(4096)]
    idx = [(i * 2654435761 + 7) % 4096 for i in range(n)]
    got = split(eng.ristretto_map_to_curve_batch(b"".join(pool32[i] for i in idx), n), 32)
    want = ho.map_to_curve_batch(pool32)
    assert all(got[i] == want[idx[i]] for i in range(n))
    got = split(eng.ristretto_lizard_encode_batch(b"".join(pool16[i] for i in idx), n), 32)
    want = ho.lizard_encode_batch(pool16)
    assert all(got[i] == want[idx[i]] for i in range(n))
    # decode and the inverse on RISTRETTO and EXTENDED input
    encs, ext = _random_points(rnd, ho, 1024)
    for fmt, pool in ((2, encs), (1, ext)):
        items = [pool[(i * 40503 + 11) % len(pool)] for i in range(n)]
        want_raw, want_st = ho.lizard_decode_batch(pool, fmt)
        want_inv, want_masks = ho.map_to_curve_inverse_batch(pool, fmt)
        rc, raw, st = eng.ristretto_lizard_decode_batch(b"".join(items), n, fmt)
        assert rc == 1
        rc2, inv, masks = eng.ristretto_map_to_curve_inverse_batch(b"".join(items), n, fmt)
        assert rc2 == 0
        for i in range(n):
            k = (i * 40503 + 11) % len(pool)
            assert st[i] == want_st[k] and raw[16 * i:16 * i + 16] == want_raw[16 * k:16 * k + 16], (fmt, i)
            assert masks[i] == want_masks[k] and inv[512 * i:512 * i + 512] == want_inv[512 * k:512 * k + 512], (fmt, i)


def test_round_trip_two_to_the_twenty(eng):
    rnd = random.Random(22)
    n = 2**20
    data = rnd.randbytes(16 * n)
    enc = eng.ristretto_lizard_encode_batch(data, n)
    rc, back, st = eng.ristretto_lizard_decode_batch(enc, n)
    assert rc == 0 and st == bytes(n) and back == data


def test_inverse_properties(eng, ho):
    rnd = random.Random(23)
    n = 4096
    ins = [rnd.randbytes(32) for _ in range(n)]
    pts = split(eng.ristretto_map_to_curve_batch(b"".join(ins), n), 32)
    rc, inv, masks = eng.ristretto_map_to_curve_inverse_batch(b"".join(pts), n)
    assert rc == 0 and all(masks)
    somes, owners = [], []
    for i in range(n):
        for j in range(16):
            if masks[i] >> j & 1:
                somes.append(inv[512 * i + 32 * j:512 * i + 32 * j + 32]); owners.append(i)
    back = split(eng.ristretto_map_to_curve_batch(b"".join(somes), len(somes)), 32)
    assert all(back[k] == pts[owners[k]] for k in range(len(somes)))
    # restricted inputs (lizard_ristretto.rs:371-406): the input appears exactly once, in the first eight slots, for the
    # representative map_to_curve returns
    for _ in range(200):
        b = bytearray(rnd.randbytes(32)); b[31] &= 0x3f; b[0] &= 0xfe; b = bytes(b)
        P = L.map_to_curve_point(b)
        rc, raw, m = eng.ristretto_map_to_curve_inverse_batch(L.limbs_bytes(P), 1, 1)
        hits = [j for j in range(16) if m[0] >> j & 1 and raw[32 * j:32 * j + 32] == b]
        assert len(hits) == 1 and hits[0] < 8


def test_decode_coset_and_scaling_invariance(eng, ho):
    rnd = random.Random(24)
    datas = [rnd.randbytes(16) for _ in range(64)]
    encs = ho.lizard_encode_batch(datas)
    items, want = [], []
    for d, e in zip(datas, encs):
        P = L.ristretto_decode(e)
        for Q in L.coset4(P):
            for lam in (1, rnd.randrange(2, L.p), rnd.randrange(2, L.p)):
                items.append(L.limbs_bytes(L.scale(Q, lam))); want.append(d)
    rc, raw, st = eng.ristretto_lizard_decode_batch(b"".join(items), len(items), 1)
    assert rc == 0 and split(raw, 16) == want


def test_undecodable_at_piece_slots(eng, golden):
    rnd = random.Random(25)
    bad = [bytes.fromhex(v["point"]) for v in golden["points"] if v["status"] == 2]
    n = 2 * PIECE + 1001
    datas = [rnd.randbytes(16) for _ in range(n)]
    encs = split(eng.ristretto_lizard_encode_batch(b"".join(datas), n), 32)
    slots = sorted({s for lo in range(0, n, PIECE) for s in (lo, lo + min(PIECE, n - lo) // 2, min(lo + PIECE, n) - 1)})
    for k, s in enumerate(slots):
        encs[s] = bad[k % len(bad)]
    rc, raw, st = eng.ristretto_lizard_decode_batch(b"".join(encs), n)
    assert rc == 1
    assert [i for i in range(n) if st[i]] == slots and all(st[s] == 2 for s in slots)
    assert all(raw[16 * s:16 * s + 16] == bytes(16) for s in slots)
    assert all(raw[16 * i:16 * i + 16] == datas[i] for i in range(n) if i not in set(slots))
    rc, inv, masks = eng.ristretto_map_to_curve_inverse_batch(b"".join(encs), n)
    assert rc == 1
    assert all(masks[s] == 0 and inv[512 * s:512 * s + 512] == bytes(512) for s in slots)
    assert all(masks[i] for i in range(0, n, 997) if i not in set(slots))


def test_elgamal_style_chain(eng, pkg):
    """mul_batch(x^-1, mul_batch(x, lizard_encode(d))) decodes to d."""
    rnd = random.Random(26)
    n = 2048
    datas = [rnd.randbytes(16) for _ in range(n)]
    xs = [rnd.randrange(1, GROUP_L) for _ in range(n)]
    enc = pkg.RistrettoPoint.lizard_encode_batch(datas, engine=eng)
    c = pkg.RistrettoPoint.mul_batch([x.to_bytes(32, "little") for x in xs], enc, engine=eng)
    back = pkg.RistrettoPoint.mul_batch([pow(x, -1, GROUP_L).to_bytes(32, "little") for x in xs], c, engine=eng)
    assert back == enc
    assert pkg.RistrettoPoint.lizard_decode_batch(back, engine=eng) == datas


def test_invalid_arguments(eng, pkg):
    lib, h = eng.lib, eng.h
    out = (C.c_uint8 * 1024)()
    st = (C.c_uint8 * 4)()
    mask = (C.c_uint16 * 4)()
    enc = pkg.RistrettoPoint.lizard_encode_batch([bytes(16)], engine=eng)[0]
    m2c, e, d, inv = (lib.dalek_b200_ristretto_map_to_curve_batch, lib.dalek_b200_ristretto_lizard_encode_batch,
                      lib.dalek_b200_ristretto_lizard_decode_batch, lib.dalek_b200_ristretto_map_to_curve_inverse_batch)
    assert m2c(h, bytes(32), 1, out) == 0 and m2c(h, None, 1, out) == -1 and m2c(h, bytes(32), 1, None) == -1
    assert m2c(h, None, 0, None) == 0
    assert e(h, bytes(16), 1, out) == 0 and e(h, None, 1, out) == -1 and e(h, bytes(16), 1, None) == -1 and e(h, None, 0, None) == 0
    for fmt in (2, 1):
        pt = enc if fmt == 2 else L.limbs_bytes(L.ristretto_decode(enc))
        assert d(h, pt, fmt, 1, out, st) == 0 and st[0] == 0
        assert d(h, None, fmt, 1, out, st) == -1 and d(h, pt, fmt, 1, None, st) == -1 and d(h, pt, fmt, 1, out, None) == -1
        assert d(h, None, fmt, 0, None, None) == 0
        assert inv(h, pt, fmt, 1, out, mask) == 0 and mask[0]
        assert inv(h, None, fmt, 1, out, mask) == -1 and inv(h, pt, fmt, 1, None, mask) == -1 and inv(h, pt, fmt, 1, out, None) == -1
        assert inv(h, None, fmt, 0, None, None) == 0
    for fmt in (0, 3, -1):                               # COMPRESSED and unknown formats
        assert d(h, enc, fmt, 1, out, st) == -1
        assert inv(h, enc, fmt, 1, out, mask) == -1
        assert d(h, None, fmt, 0, None, None) == -1
    assert pkg.RistrettoPoint.lizard_encode_batch([], engine=eng) == []
    assert pkg.RistrettoPoint.lizard_decode_batch([], engine=eng) == []
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.lizard_encode_batch([bytes(15)], engine=eng)


def test_last_call_ms_covers_the_calls(eng):
    rnd = random.Random(27)
    enc = eng.ristretto_lizard_encode_batch(rnd.randbytes(16 * 1000), 1000)
    assert eng.last_call_ms() > 0
    eng.ristretto_lizard_decode_batch(enc, 1000)
    assert eng.last_call_ms() > 0
