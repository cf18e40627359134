"""GPU batched independent MSMs: dalek_b200_msm_batch / _dev (m MSMs, each with its own scalars and points, in one
call; variable time and constant time; Edwards and Ristretto) against the C oracle, the single-MSM entry points and the
algebraic identity sum s_i (t_i B) = (sum s_i t_i) B."""
import array
import json
import os
import random

import pytest

import msm_digit_cases
import oracle_lib
import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
OK, DALEK_NONE = 0, 1
LARGE_MIN = 1 << 15                               # msm_batch.cu MB_LARGE_MIN
PIECE_TERMS = 1 << 18                             # msm_batch.cu MB_PIECE_TERMS
SIZES = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 189, 190, 250, 499, 500, 1000]
FORMATS = [COMPRESSED, EXTENDED, RISTRETTO]


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
def pool(orc):
    """64 prime-order points: (oracle point, {format: input bytes})"""
    rnd = random.Random(2024)
    B = orc.basepoint()
    return [with_inputs(orc, orc.scalarmul(b32(rnd.randrange(1, L)), B)) for _ in range(64)]


def b32(x):
    return x.to_bytes(32, "little")


def with_inputs(orc, P):
    return P, {COMPRESSED: orc.compress(P), RISTRETTO: orc.ristretto_compress(P),
               EXTENDED: b"".join(int(v).to_bytes(8, "little") for v in orc.p3_limbs(P))}


def encode(orc, P, fmt):
    return orc.ristretto_compress(P) if fmt == RISTRETTO else orc.compress(P)


def identity_enc(fmt):
    return bytes(32) if fmt == RISTRETTO else b32(1)


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf) or bytearray(8), dtype=torch.uint8).cuda()


def offsets_of(sizes):
    offs = array.array("Q", [0])
    for n in sizes:
        offs.append(offs[-1] + n)
    return offs


def run(eng, segs, fmt, ct, device=False, want_limbs=False, point_bytes=None):
    """segs: list of (scalars, pool entries).  Returns (rc, [32-byte outputs], ok bytes, limbs or None)."""
    flat_s = b"".join(b"".join(s) for s, _ in segs)
    flat_p = b"".join(point_bytes) if point_bytes is not None else b"".join(p[1][fmt] for _, ps in segs for p in ps)
    offs = offsets_of([len(s) for s, _ in segs]).tobytes()
    if device:
        rc, out, ok, limbs = eng.msm_batch(dev(flat_s), dev(flat_p), dev(offs), len(segs), fmt, constant_time=ct, device_ptrs=True,
                                           want_limbs=want_limbs)
    else:
        rc, out, ok, limbs = eng.msm_batch(flat_s, flat_p, offs, len(segs), fmt, constant_time=ct, want_limbs=want_limbs)
    return rc, [out[32 * j:32 * j + 32] for j in range(len(segs))], ok, limbs


def oracle_seg(orc, scalars, entries, fmt, ct):
    pts = [e[0] for e in entries]
    return encode(orc, orc.msm_ct(scalars, pts) if ct else orc.msm("optional", scalars, pts), fmt)


def random_segs(rnd, pool, sizes, top=L):
    return [([b32(rnd.randrange(top)) for _ in range(n)], [pool[rnd.randrange(len(pool))] for _ in range(n)]) for n in sizes]


@pytest.mark.parametrize("ct", [False, True])
@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_parity_per_segment(eng, orc, pool, fmt, ct):
    rnd = random.Random(31 + fmt + 10 * ct)
    sizes = SIZES + [LARGE_MIN + 5]
    rnd.shuffle(sizes)
    segs = random_segs(rnd, pool, sizes, top=2**255 if ct else L)
    rc, out, ok, _ = run(eng, segs, fmt, ct)
    assert rc == OK and ok == b"\x01" * len(segs)
    for (s, ps), got in zip(segs, out):
        assert got == oracle_seg(orc, s, ps, fmt, ct), len(s)


def test_equal_to_the_single_calls(eng, orc, pool):
    rnd = random.Random(41)
    sizes = [0, 1, 2, 5, 16, 17, 64, 189, 190, 300, 1000, LARGE_MIN]
    segs = random_segs(rnd, pool, sizes)
    for fmt in (COMPRESSED, EXTENDED):
        for ct in (False, True):
            rc, out, _, limbs = run(eng, segs, fmt, ct, want_limbs=True)
            assert rc == OK
            for j, (s, ps) in enumerate(segs):
                pts = b"".join(p[1][fmt] for p in ps)
                single = eng.edwards_ct_msm if ct else eng.edwards_vartime_msm
                rc1, comp, lb = single(b"".join(s), pts, len(s), point_fmt=fmt, want_limbs=True)
                assert rc1 == OK and comp == out[j], (fmt, ct, len(s))
                assert orc.ct_eq(orc.p3_from_limbs(lb), orc.p3_from_limbs(limbs[20 * j:20 * j + 20]))
                assert orc.compress(orc.p3_from_limbs(limbs[20 * j:20 * j + 20])) == out[j]
    rc, out, _, _ = run(eng, segs, RISTRETTO, False)
    for j, (s, ps) in enumerate(segs):
        assert eng.ristretto_vartime_msm(b"".join(s), b"".join(p[1][RISTRETTO] for p in ps), len(s)) == (OK, out[j])


def test_constant_time_ristretto_pairs_equal_double_base_batch(eng, pool):
    rnd = random.Random(42)
    G, H = pool[3], pool[4]
    n = 100
    a, b = [b32(rnd.randrange(L)) for _ in range(n)], [b32(rnd.randrange(L)) for _ in range(n)]
    rc, out, ok, _ = run(eng, [([x, y], [G, H]) for x, y in zip(a, b)], RISTRETTO, True)
    rc2, want = eng.ristretto_double_base_batch(b"".join(a), b"".join(b), G[1][RISTRETTO], H[1][RISTRETTO], n)
    assert rc == rc2 == OK and b"".join(out) == want


@pytest.mark.parametrize("ct", [False, True])
def test_edge_scalars_and_digit_boundaries(eng, orc, pool, ct):
    vals = [s for c in (4, 5, 13) for s in msm_digit_cases.boundary_scalars(c) if s < 2**255]
    vals += [0, 1, L - 1, L, 2**255 - 1]
    segs = [([b32(s)], [pool[i % 64]]) for i, s in enumerate(vals)]
    segs += [([b32(s) for s in vals[lo:lo + 21]], [pool[(lo + k) % 64] for k in range(len(vals[lo:lo + 21]))]) for lo in range(0, len(vals), 21)]
    rc, out, _, _ = run(eng, segs, COMPRESSED, ct)
    assert rc == OK
    for (s, ps), got in zip(segs, out):
        assert got == oracle_seg(orc, s, ps, COMPRESSED, ct)


def test_scalar_with_bit_255_set_behaves_as_the_single_call(eng, pool):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(43)
    segs = [([b32(2**255), b32(2**256 - 1), b32(rnd.randrange(2**255, 2**256))], pool[:3]), ([b32(2**255 + 7)], pool[5:6])]
    rc, out, _, _ = run(eng, segs, COMPRESSED, False)
    assert rc == OK
    for (s, ps), got in zip(segs, out):
        assert eng.edwards_vartime_msm(b"".join(s), b"".join(p[1][COMPRESSED] for p in ps), len(s))[:2] == (OK, got)
    for device in (False, True):
        with pytest.raises(pkg.EngineError):
            run(eng, segs, COMPRESSED, True, device=device)
    with pytest.raises(pkg.EngineError):
        eng.edwards_ct_msm(b"".join(segs[1][0]), pool[5][1][COMPRESSED], 1)


@pytest.mark.parametrize("ct", [False, True])
def test_identity_torsion_cancellation_and_repeated_points(eng, orc, pool, ct):
    rnd = random.Random(44)
    ident = with_inputs(orc, orc.identity())
    tors = [with_inputs(orc, t) for t in torsion_points(orc)]
    mixed = [with_inputs(orc, orc.add(pool[i][0], t[0])) for i, t in enumerate(tors)]
    s = rnd.randrange(L)
    segs = [([b32(rnd.randrange(L))], [ident]), ([b32(3), b32(5), b32(0)], [ident, pool[0], ident])]
    segs += [([b32(k)], [t]) for t in tors for k in (1, 7, 8, rnd.randrange(L))]
    segs += [([b32(rnd.randrange(L)) for _ in range(7)], tors), ([b32(rnd.randrange(L)) for _ in range(7)], mixed)]
    segs += [([b32(rnd.randrange(L)) for _ in range(14)], tors + mixed)]
    segs += [([b32(s), b32(L - s)], [pool[1], pool[1]])]                       # cancels to the identity
    segs += [([b32(s), b32(7), b32(L - s), b32(L - 7)], [pool[1], pool[2], pool[1], pool[2]])]
    segs += [([b32(s)] * 5, [pool[9]] * 5)]                                    # equal accumulator and addend: a doubling
    segs += [([b32(1), b32(1), b32(2)], [pool[9]] * 3)]
    for fmt in (COMPRESSED, EXTENDED):
        rc, out, _, _ = run(eng, segs, fmt, ct)
        assert rc == OK
        for (sc, ps), got in zip(segs, out):
            assert got == oracle_seg(orc, sc, ps, fmt, ct)
    assert out[-4] == out[-3] == b32(1)


def ristretto_bad():
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        return bytes.fromhex(json.load(f)["classes"]["nonsquare"][0]["s"])


@pytest.mark.parametrize("fmt,bad", [(COMPRESSED, b32(2)), (RISTRETTO, None)])
def test_none_is_per_segment(eng, orc, pool, fmt, bad):
    import curve25519_dalek_b200 as pkg
    bad = bad or ristretto_bad()
    rnd = random.Random(45)
    sizes = [40, 3, 0, 17, 40, 1, 40, 64]
    segs = random_segs(rnd, pool, sizes)
    rc, clean, ok, _ = run(eng, segs, fmt, False)
    assert rc == OK and ok == b"\x01" * len(sizes)
    starts = offsets_of(sizes)
    pts = [p[1][fmt] for _, ps in segs for p in ps]
    for seg, at in ((0, 0), (4, 39), (6, 21), (5, 0)):                      # first, last, mid-chunk, a one-term MSM
        broken = list(pts)
        broken[starts[seg] + at] = bad
        rc, out, ok, _ = run(eng, segs, fmt, False, point_bytes=broken)
        assert rc == DALEK_NONE
        assert ok == bytes(0 if j == seg else 1 for j in range(len(sizes)))
        assert out == [identity_enc(fmt) if j == seg else clean[j] for j in range(len(sizes))]
        rc, out_d, ok_d, _ = run(eng, segs, fmt, False, device=True, point_bytes=broken)
        assert (rc, out_d, ok_d) == (DALEK_NONE, out, ok)
        with pytest.raises(pkg.EngineError):
            run(eng, segs, fmt, True, point_bytes=broken)


def test_argument_errors_and_empty_calls(eng, pool):
    import curve25519_dalek_b200 as pkg
    s, p = b32(5) * 4, pool[0][1][COMPRESSED] * 4
    for offs in ([1, 2, 4], [0, 3, 2], [0, 2, 2**31], [0, 2**40, 2**41]):
        with pytest.raises(pkg.EngineError):
            eng.msm_batch(s, p, array.array("Q", offs).tobytes(), 2)
    good = array.array("Q", [0, 2, 4]).tobytes()
    with pytest.raises(pkg.EngineError):
        eng.msm_batch(s, p, good, 2, point_fmt=7)
    for args in ((None, p, good), (s, None, good), (s, p, None)):
        with pytest.raises(pkg.EngineError):
            eng.msm_batch(*args, 2)
    assert eng.msm_batch(None, None, None, 0)[:3] == (OK, b"", b"")
    for fmt in FORMATS:
        for ct in (False, True):
            rc, out, ok, limbs = eng.msm_batch(None, None, array.array("Q", [0] * 6).tobytes(), 5, fmt, constant_time=ct, want_limbs=True)
            assert (rc, out, ok) == (OK, identity_enc(fmt) * 5, b"\x01" * 5)
            assert limbs == ([0] * 5 + [1] + [0] * 4 + [1] + [0] * 9) * 5


@pytest.mark.parametrize("ct", [False, True])
def test_device_pointers_give_the_same_bytes(eng, pool, ct):
    rnd = random.Random(46)
    segs = random_segs(rnd, pool, [0, 1, 33, 500, 16, 0, 250, 2])
    for fmt in FORMATS:
        assert run(eng, segs, fmt, ct, device=True, want_limbs=True) == run(eng, segs, fmt, ct, want_limbs=True)


def algebraic_batch(eng, rnd, sizes):
    """points t_i B from the engine, scalars s_i: per MSM the expected encoding of (sum s_i t_i) B"""
    total = sum(sizes)
    t = [rnd.randrange(L) for _ in range(total)]
    s = [rnd.randrange(L) for _ in range(total)]
    limbs, comp = eng.mul_base_batch(b"".join(map(b32, t)), total)
    want, at = [], 0
    for n in sizes:
        want.append(sum(a * b for a, b in zip(s[at:at + n], t[at:at + n])) % L)
        at += n
    _, expect = eng.mul_base_batch(b"".join(map(b32, want)), len(sizes))
    return b"".join(map(b32, s)), comp, bytes(limbs), expect


@pytest.mark.parametrize("ct", [False, True])
def test_piece_boundaries(eng, ct):
    """More terms than one piece holds, with an MSM across the place where a cut by term count alone would fall."""
    rnd = random.Random(47)
    sizes = [1000] * 260 + [PIECE_TERMS - 260000 - 10, 20, 3000, 1, 0, 7]      # the 20-term MSM straddles PIECE_TERMS
    sizes += [PIECE_TERMS + 3] if ct else [LARGE_MIN - 1] * 6                  # constant time: an MSM larger than a piece
    s, comp, _, expect = algebraic_batch(eng, rnd, sizes)
    rc, out, ok, _ = eng.msm_batch(s, comp, offsets_of(sizes).tobytes(), len(sizes), constant_time=ct)
    assert rc == OK and ok == b"\x01" * len(sizes) and out == expect


@pytest.mark.parametrize("sizes", [[256] * 4096, [4] * (1 << 18)], ids=["4096x256", "262144x4"])
def test_scale(eng, orc, sizes):
    rnd = random.Random(48)
    s, comp, limbs, expect = algebraic_batch(eng, rnd, sizes)
    offs = offsets_of(sizes)
    m = len(sizes)
    rc, out, ok, _ = eng.msm_batch(s, comp, offs.tobytes(), m)
    assert rc == OK and ok == b"\x01" * m and out == expect
    assert eng.msm_batch(s, limbs, offs.tobytes(), m, EXTENDED, constant_time=True)[:3] == (OK, expect, ok)
    for j in rnd.sample(range(m), 64):
        lo, hi = offs[j], offs[j + 1]
        pts = [orc.decompress(comp[32 * i:32 * i + 32]) for i in range(lo, hi)]
        assert orc.compress(orc.msm("optional", [s[32 * i:32 * i + 32] for i in range(lo, hi)], pts)) == out[32 * j:32 * j + 32]


def test_trait_style_methods(eng, orc, pool):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(49)
    segs = random_segs(rnd, pool, [3, 0, 20])
    for cls, fmt in ((pkg.EdwardsPoint, COMPRESSED), (pkg.RistrettoPoint, RISTRETTO)):
        sl, plist = [s for s, _ in segs], [[p[1][fmt] for p in ps] for _, ps in segs]
        want = [oracle_seg(orc, s, ps, fmt, False) for s, ps in segs]
        assert cls.optional_multiscalar_mul_batch(sl, plist, engine=eng) == want
        assert cls.vartime_multiscalar_mul_batch(sl, plist, engine=eng) == want
        assert cls.multiscalar_mul_batch(sl, plist, engine=eng) == want
        broken = [list(p) for p in plist]
        broken[0][1] = None
        broken[2][19] = b32(2) if fmt == COMPRESSED else ristretto_bad()
        assert cls.optional_multiscalar_mul_batch(sl, broken, engine=eng) == [None, want[1], None]
        with pytest.raises(ValueError):
            cls.vartime_multiscalar_mul_batch(sl, broken, engine=eng)
        with pytest.raises(AssertionError):
            cls.optional_multiscalar_mul_batch([sl[0][:2]], [plist[0]], engine=eng)
