"""Hashing into the group on the GPU: every golden vector through every entry point (C ABI and module-level Python),
random parity with the C oracle across piece boundaries, mixed message lengths, the D = 0 and boundary halves at the
first, middle and last slot of a piece, generator derivation feeding precomputations and MSMs, and argument checks."""
import ctypes as C
import json
import os
import random

import pytest

import h2c_oracle
import oracle_lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = 2**252 + 27742317777372353535851937790883648493


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
    with open(os.path.join(ROOT, "tests", "golden", "hash_to_curve.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def ho():
    return h2c_oracle.load()


def flat(msgs):
    offs = (C.c_uint64 * (len(msgs) + 1))()
    acc = 0
    for i, m in enumerate(msgs):
        offs[i] = acc
        acc += len(m)
    offs[len(msgs)] = acc
    return b"".join(msgs) + b"\0", offs


def split(raw):
    return [raw[i:i + 32] for i in range(0, len(raw), 32)]


def run(eng, kind, items, dst=b"x"):
    """One C-ABI batch: kind in from_uniform | hash_from_bytes | hash_to_curve | encode_to_curve."""
    if kind == "from_uniform":
        return split(eng.ristretto_from_uniform_bytes_batch(b"".join(items), len(items)))
    buf, offs = flat(items)
    if kind == "hash_from_bytes":
        return split(eng.ristretto_hash_from_bytes_batch(buf, offs, len(items)))
    fn = eng.edwards_hash_to_curve_batch if kind == "hash_to_curve" else eng.edwards_encode_to_curve_batch
    return split(fn(buf, offs, len(items), dst))


def oracle(ho, kind, items, dst=b"x"):
    if kind == "from_uniform":
        return ho.from_uniform_batch(items)
    return ho.flat_batch(kind, items, dst)


def test_golden_vectors_c_abi_and_python(eng, pkg, golden):
    ro, nu = bytes.fromhex(golden["dst_ro"]), bytes.fromhex(golden["dst_nu"])
    ins = [bytes.fromhex(v["in"]) for v in golden["one_way_map"] + golden["from_uniform_edges"]]
    outs = [v["out"] for v in golden["one_way_map"] + golden["from_uniform_edges"]]
    assert [x.hex() for x in run(eng, "from_uniform", ins)] == outs
    assert [x.hex() for x in pkg.RistrettoPoint.from_uniform_bytes_batch(ins, engine=eng)] == outs
    msgs = [bytes.fromhex(v["msg"]) for v in golden["hash_from_bytes_lengths"]]
    want = [v["out"] for v in golden["hash_from_bytes_lengths"]]
    assert [x.hex() for x in run(eng, "hash_from_bytes", msgs)] == want
    assert [x.hex() for x in pkg.RistrettoPoint.hash_from_bytes_batch(msgs, engine=eng)] == want
    for key, dst, kind, pyfn in (("rfc9380_hash_to_curve", ro, "hash_to_curve", pkg.EdwardsPoint.hash_to_curve_batch),
                                 ("rfc9380_encode_to_curve", nu, "encode_to_curve", pkg.EdwardsPoint.encode_to_curve_batch)):
        msgs = [bytes.fromhex(v["msg"]) for v in golden[key]]
        want = [v["out"] for v in golden[key]]
        assert [x.hex() for x in run(eng, kind, msgs, dst)] == want
        assert [x.hex() for x in pyfn(msgs, dst, engine=eng)] == want
    # XMD block and DST boundaries: one batch per DST
    by_dst = {}
    for v in golden["xmd_boundaries"]:
        by_dst.setdefault(v["dst"], []).append(v)
    for dh, vs in by_dst.items():
        dst = bytes.fromhex(dh)
        msgs = [bytes.fromhex(v["msg"]) for v in vs]
        assert [x.hex() for x in run(eng, "hash_to_curve", msgs, dst)] == [v["hash_to_curve"] for v in vs]
        assert [x.hex() for x in pkg.EdwardsPoint.encode_to_curve_batch(msgs, dst, engine=eng)] == [v["encode_to_curve"] for v in vs]


@pytest.mark.parametrize("kind", ["from_uniform", "hash_from_bytes", "hash_to_curve", "encode_to_curve"])
def test_random_parity_across_piece_sizes(eng, ho, kind):
    rnd = random.Random(hash(kind) & 0xffff)
    dst = rnd.randbytes(rnd.randrange(1, 256))
    big = 2**17 + 3
    pool = [rnd.randbytes(64) if kind == "from_uniform" else rnd.randbytes(rnd.randrange(0, 80)) for _ in range(4096)]
    want_pool = oracle(ho, kind, pool, dst)
    for n in (1, 7, 8, 9, 127, 128, 129, 2**16 - 1, 2**16, 2**16 + 1, big):
        idx = [(i * 2654435761 + n) % len(pool) for i in range(n)]
        got = run(eng, kind, [pool[i] for i in idx], dst)
        assert len(got) == n
        bad = [i for i in range(n) if got[i] != want_pool[idx[i]]]
        assert not bad, (n, bad[:5])


def test_mixed_lengths_in_one_batch(eng, ho):
    rnd = random.Random(7)
    msgs = [rnd.randbytes(k) for k in range(401)]
    msgs += [b"", msgs[300], b"", msgs[5], msgs[400]]
    rnd.shuffle(msgs)
    for kind in ("hash_from_bytes", "hash_to_curve", "encode_to_curve"):
        dst = b"mixed-" + kind.encode()
        assert run(eng, kind, msgs, dst) == oracle(ho, kind, msgs, dst), kind


def test_d_zero_and_boundary_halves_at_piece_slots(eng, ho, golden):
    rnd = random.Random(8)
    specials = [bytes.fromhex(v["in"]) for v in golden["from_uniform_edges"]]
    for n in (300, 2**17 + 3):
        items = [rnd.randbytes(64) for _ in range(n)]
        piece = 2**16 if n >= 2**17 else n
        slots = sorted({s for lo in range(0, n, piece) for s in (lo, lo + min(piece, n - lo) // 2, min(lo + piece, n) - 1)})
        for k, s in enumerate(slots):
            items[s] = specials[k % len(specials)]
        got = run(eng, "from_uniform", items)
        for s in slots:
            assert got[s] == ho.from_uniform_bytes(items[s]), s
        for s in rnd.sample(range(n), 64):
            assert got[s] == ho.from_uniform_bytes(items[s])


def test_generators_feed_precomputation_and_msm(eng, pkg, ho):
    orc = oracle_lib.load()
    rnd = random.Random(9)
    n = 4096
    labels = [b"gen-%d" % i for i in range(n)]
    scalars = [rnd.randrange(L).to_bytes(32, "little") for _ in range(n)]
    dst = b"generator-derivation-test"
    cases = [
        ("from_uniform", [rnd.randbytes(64) for _ in range(n)], True),
        ("hash_from_bytes", labels, True),
        ("hash_to_curve", labels, False),
        ("encode_to_curve", labels, False),
    ]
    for kind, items, ristretto in cases:
        gens = run(eng, kind, items, dst)
        want_gens = oracle(ho, kind, items, dst)
        assert gens == want_gens, kind
        if ristretto:
            pre = pkg.VartimeRistrettoPrecomputation(gens, engine=eng)
            pts = [orc.ristretto_decompress(g) for g in want_gens]
            want = orc.ristretto_compress(orc.msm("optional", scalars, pts))
        else:
            pre = pkg.VartimeEdwardsPrecomputation(gens, engine=eng)
            pts = [orc.decompress(g) for g in want_gens]
            want = orc.compress(orc.msm("optional", scalars, pts))
        assert pre.vartime_multiscalar_mul(scalars) == want, kind
        pre.close()
        if not ristretto:
            rc, got, _ = eng.edwards_vartime_msm(b"".join(scalars), b"".join(gens), n)
            assert rc == 0 and got == want


def test_invalid_arguments(eng):
    lib, h = eng.lib, eng.h
    buf, offs = flat([b"ab", b"c"])
    out = (C.c_uint8 * 64)()
    dst = b"dst"
    h2c = lib.dalek_b200_edwards_hash_to_curve_batch
    e2c = lib.dalek_b200_edwards_encode_to_curve_batch
    for fn in (h2c, e2c):
        assert fn(h, buf, offs, 2, dst, 3, out) == 0
        assert fn(h, buf, offs, 2, dst, 0, out) == -1
        assert fn(h, buf, offs, 2, b"d" * 256, 256, out) == -1
        assert fn(h, buf, offs, 2, b"d" * 255, 255, out) == 0
        assert fn(h, buf, offs, 2, None, 3, out) == -1
        assert fn(h, None, offs, 2, dst, 3, out) == -1
        assert fn(h, buf, None, 2, dst, 3, out) == -1
        assert fn(h, buf, offs, 2, dst, 3, None) == -1
        assert fn(h, None, None, 0, dst, 3, None) == 0
    hfb = lib.dalek_b200_ristretto_hash_from_bytes_batch
    assert hfb(h, buf, offs, 2, out) == 0
    assert hfb(h, None, offs, 2, out) == -1 and hfb(h, buf, None, 2, out) == -1 and hfb(h, buf, offs, 2, None) == -1
    assert hfb(h, None, None, 0, None) == 0
    dec = (C.c_uint64 * 3)(0, 2, 1)
    nz = (C.c_uint64 * 3)(1, 2, 3)
    for o in (dec, nz):
        assert hfb(h, buf, o, 2, out) == -1
        assert h2c(h, buf, o, 2, dst, 3, out) == -1
        assert e2c(h, buf, o, 2, dst, 3, out) == -1
    fub = lib.dalek_b200_ristretto_from_uniform_bytes_batch
    assert fub(h, None, 1, out) == -1 and fub(h, bytes(64), 1, None) == -1 and fub(h, None, 0, None) == 0
    assert fub(h, bytes(64), 1, out) == 0


def test_last_call_ms_covers_the_calls(eng):
    rnd = random.Random(10)
    eng.ristretto_from_uniform_bytes_batch(rnd.randbytes(64 * 1000), 1000)
    assert eng.last_call_ms() > 0
    buf, offs = flat([rnd.randbytes(32) for _ in range(1000)])
    eng.edwards_hash_to_curve_batch(buf, offs, 1000, b"t")
    assert eng.last_call_ms() > 0
