"""Every extended point an entry point of include/dalek_b200.h returns as limbs is a valid EdwardsPoint
(tests/point_checks.py): limbs < 2^51, coordinates < p, Z != 0, X Y = Z T, on the curve, and projectively the oracle's
point.  Comparing encodings alone would not notice a wrong T: compression ignores it, but a caller who adds to the
returned point reads it.  Edge results too: n = 0, the identity, small-order results and an all-even Straus warp."""
import array
import ctypes as C
import random

import pytest

import point_checks
import pyref
import straus_patterns as sp

pytestmark = pytest.mark.gpu

COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf) or bytearray(8), dtype=torch.uint8).cuda()


def b32(v):
    return v.to_bytes(32, "little")


def cases(oracle):
    """(name, integer scalars, oracle points): the edge results and both MSM paths"""
    rnd = random.Random(4242)
    pts = sp.random_points(oracle, rnd, 300)
    small = sp.small_order_points(oracle)
    return [
        ("empty", [], []),
        ("identity_result", [0] * 12, pts[:12]),
        ("identity_result_L", [pyref.L] * 3, pts[:3]),
        ("small_order_result", [1, 3, 5, 7], small),
        ("all_even_warp", sp.pattern_scalars("even", rnd, 8), pts[:8]),
        ("all_even_warps_with_small_order", sp.layout(20, {}, "even", rnd), pts[:16] + small),
        ("straus_random", [rnd.randrange(pyref.L) for _ in range(100)], pts[:100]),
        ("bucket_random", [rnd.randrange(pyref.L) for _ in range(300)], pts),
    ]


def ext_limbs(oracle, P):
    q = oracle.sub(oracle.add(oracle.double(P), P), oracle.double(P))             # the same point, Z != 1
    return b"".join(int(v).to_bytes(8, "little") for v in oracle.p3_limbs(q))


def test_vartime_and_ct_msm_limbs(eng, oracle):
    """edwards_vartime_msm (Straus and bucket path, host and device buffers) and edwards_ct_msm."""
    for name, s, P in cases(oracle):
        n = len(s)
        want = oracle.compress(sp.msm_exact(oracle, s, P) if n else oracle.identity())
        sb = b"".join(b32(v) for v in s)
        comp = b"".join(oracle.compress(x) for x in P)
        ext = b"".join(ext_limbs(oracle, x) for x in P)
        for straus in (1, 0):
            eng.set_option("small_straus", straus)
            try:
                for fmt, buf in ((COMPRESSED, comp), (EXTENDED, ext)):
                    rc, got, limbs = eng.edwards_vartime_msm(sb, buf, n, point_fmt=fmt, want_limbs=True)
                    assert rc == 0 and got == want, (name, straus, fmt)
                    point_checks.check_limbs(limbs, want, what=(name, straus, fmt))
                    rc, got, limbs = eng.edwards_vartime_msm(dev(sb), dev(buf), n, point_fmt=fmt, device_ptrs=True, want_limbs=True)
                    assert rc == 0 and got == want, (name, straus, fmt, "dev")
                    point_checks.check_limbs(limbs, want, what=(name, straus, fmt, "dev"))
            finally:
                eng.set_option("small_straus", 1)
        if all(v < 1 << 255 for v in s):                          # the constant-time contract's scalars
            rc, got, limbs = eng.edwards_ct_msm(sb, comp, n, want_limbs=True)
            assert rc == 0 and got == want, (name, "ct")
            point_checks.check_limbs(limbs, want, what=(name, "ct"))


def window_digits(v, c, nwin):
    return [(v >> (c * w)) & ((1 << c) - 1) for w in range(nwin)]


@pytest.mark.parametrize("c", [5, 8, 13])
def test_partial_window_accumulators_and_combine(eng, oracle, c):
    """edwards_msm_partial: each window accumulator is a valid point (its limbs need not be canonical) and equals
    sum_i d_iw P_i -- scalars built from digits below 2^(c-1), so that no signed recoding carries.  Then
    edwards_msm_combine and _combine_dev of two such shards return valid canonical limbs of the whole MSM."""
    rnd = random.Random(c)
    eng.set_option("window_bits", c)
    try:
        n_shard = 40
        nwin = eng.msm_window_count(n_shard)
        assert nwin == 256 // c + 1
        shards = []
        for r in range(2):
            P = sp.random_points(oracle, rnd, n_shard)
            if r == 1:
                P[:4] = sp.small_order_points(oracle)
            digits = [[rnd.randrange(1 << (c - 1)) for _ in range(nwin)] for _ in range(n_shard)]
            for d in digits:                                        # keep the scalar below 2^255
                top = 255 - c * (nwin - 1)
                d[-1] &= (1 << max(top, 0)) - 1
            s = [sum(d[w] << (c * w) for w in range(nwin)) for d in digits]
            shards.append((s, P, digits))
        allw = (C.c_uint64 * (20 * nwin * 2))()
        for r, (s, P, digits) in enumerate(shards):
            rc, w = eng.edwards_msm_partial(b"".join(b32(v) for v in s), b"".join(oracle.compress(x) for x in P), n_shard, n_shard)
            assert rc == 0
            for k in range(nwin):
                want = oracle.compress(oracle.msm("straus_vartime", [b32(d[k]) for d in digits], P))
                point_checks.check_limbs(list(w[20 * k:20 * k + 20]), want, canonical=False, what=("window", r, k))
            for k in range(20 * nwin):
                allw[r * 20 * nwin + k] = w[k]
        s_all = shards[0][0] + shards[1][0]
        want = oracle.compress(oracle.msm("optional", [b32(v) for v in s_all], shards[0][1] + shards[1][1]))
        got, limbs = eng.edwards_msm_combine(allw, 2, n_shard, want_limbs=True)
        assert got == want
        point_checks.check_limbs(limbs, want, what="combine")
        rec = eng.msm_partial_bytes(n_shard)
        import torch
        gathered = torch.zeros(2 * rec, dtype=torch.uint8, device="cuda")
        for r, (s, P, _) in enumerate(shards):
            assert eng.edwards_msm_partial_async(b"".join(b32(v) for v in s), b"".join(oracle.compress(x) for x in P), n_shard, n_shard,
                                                 gathered.data_ptr() + r * rec) == 0
        rc, got, limbs = eng.edwards_msm_combine_dev(gathered.data_ptr(), 2, n_shard, want_limbs=True)
        assert rc == 0 and got == want
        point_checks.check_limbs(limbs, want, what="combine_dev")
    finally:
        eng.set_option("window_bits", 0)


def test_precomp_mixed_msm_limbs(eng, oracle):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(7)
    static = sp.random_points(oracle, rnd, 30)
    dyn = sp.random_points(oracle, rnd, 8)
    pre = pkg.VartimeEdwardsPrecomputation([oracle.compress(x) for x in static], engine=eng)
    try:
        for ns, ds in ((30, sp.pattern_scalars("even", rnd, 8)), (30, []), (0, [rnd.randrange(pyref.L) for _ in range(8)]),
                       (12, [0] * 8)):
            ss = [rnd.randrange(pyref.L) & ~1 for _ in range(ns)]
            want = oracle.compress(oracle.msm("optional", [b32(v) for v in ss + ds], static[:ns] + dyn[:len(ds)])
                                   if ns + len(ds) else oracle.identity())
            out = (C.c_uint8 * 32)()
            limbs = (C.c_uint64 * 20)()
            sb, db = b"".join(b32(v) for v in ss), b"".join(b32(v) for v in ds)
            pb = b"".join(oracle.compress(x) for x in dyn[:len(ds)])
            rc = eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, sb if ns else None, ns, db if ds else None,
                                                      pb if ds else None, COMPRESSED, len(ds), C.addressof(out), C.addressof(limbs))
            assert rc == 0 and bytes(out) == want, (ns, len(ds))
            point_checks.check_limbs(list(limbs), want, what=("precomp", ns, len(ds)))
    finally:
        pre.close()


@pytest.mark.parametrize("ct", [False, True])
@pytest.mark.parametrize("device", [False, True])
def test_msm_batch_limbs(eng, oracle, ct, device):
    segs = [(s, P) for _, s, P in cases(oracle) if not ct or all(v < 1 << 255 for v in s)]
    flat_s = b"".join(b32(v) for s, _ in segs for v in s)
    flat_p = b"".join(oracle.compress(x) for _, P in segs for x in P)
    offs = array.array("Q", [0])
    for s, _ in segs:
        offs.append(offs[-1] + len(s))
    offs = offs.tobytes()
    if device:
        rc, out, ok, limbs = eng.msm_batch(dev(flat_s), dev(flat_p), dev(offs), len(segs), constant_time=ct, device_ptrs=True, want_limbs=True)
    else:
        rc, out, ok, limbs = eng.msm_batch(flat_s, flat_p, offs, len(segs), constant_time=ct, want_limbs=True)
    assert rc == 0 and ok == b"\x01" * len(segs)
    wants = [oracle.compress(sp.msm_exact(oracle, s, P) if s else oracle.identity()) for s, P in segs]
    assert [out[32 * j:32 * j + 32] for j in range(len(segs))] == wants
    point_checks.check_limb_array(limbs, wants, what=("msm_batch", ct, device))


def test_decompress_batch_limbs(eng, oracle):
    rnd = random.Random(11)
    pts = sp.random_points(oracle, rnd, 40) + sp.small_order_points(oracle)
    encs = [oracle.compress(x) for x in pts] + [b32(2), b32(pyref.p + 1), rnd.randbytes(32), rnd.randbytes(32)]
    rc, limbs, ok = eng.decompress_batch(b"".join(encs), len(encs))
    wants = []
    for e in encs:
        q = oracle.decompress(e)
        wants.append(None if q is None else oracle.compress(q))
    assert ok == bytes(int(w is not None) for w in wants)
    point_checks.check_limb_array(list(limbs), wants, what="edwards_decompress")
    renc = [oracle.ristretto_compress(x) for x in sp.random_points(oracle, rnd, 40)] + [bytes(32), b32(1), rnd.randbytes(32)]
    rc, limbs, ok = eng.decompress_batch(b"".join(renc), len(renc), ristretto=True)
    wants = []
    for e in renc:
        q = oracle.ristretto_decompress(e)
        wants.append(None if q is None else oracle.compress(q))
    assert ok == bytes(int(w is not None) for w in wants)
    point_checks.check_limb_array(list(limbs), wants, what="ristretto_decompress")


def test_mul_base_batch_limbs(eng, oracle):
    rnd = random.Random(13)
    s = [0, 1, 2, pyref.L - 1] + [rnd.randrange(pyref.L) for _ in range(60)] + [rnd.randrange(pyref.L) & ~((1 << 64) - 1) for _ in range(4)]
    limbs, comp = eng.mul_base_batch(b"".join(b32(v) for v in s), len(s))
    B = oracle.basepoint()
    wants = [oracle.compress(oracle.scalarmul(b32(v), B)) for v in s]
    assert [comp[32 * i:32 * i + 32] for i in range(len(s))] == wants
    point_checks.check_limb_array(list(limbs), wants, what="mul_base")
