"""GPU parity tests for VartimePrecomputedMultiscalarMul (C/traits.rs:290-406; VartimeEdwardsPrecomputation
C/edwards.rs:1038-1076, VartimeRistrettoPrecomputation C/ristretto.rs:1004-1049) against the CPU oracle.
Mirrors the reference's own tests `vartime_precomputed_vs_nonprecomputed_multiscalar` (C/edwards.rs:2343-2417)
and `mixed_multiscalar` style checks: the precomputed result equals the plain MSM over the concatenated terms."""
import ctypes as C
import random

import pytest

import pyref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    tables = e.get_option("precomp_tables")
    yield e
    assert e.get_option("precomp_tables") == tables        # no test leaves the option changed
    e.close()


def b32(x):
    return x.to_bytes(32, "little")


def rand_points(oracle, rnd, n):
    B = oracle.basepoint()
    return [oracle.scalarmul(b32(rnd.randrange(pyref.L)), B) for _ in range(n)]


@pytest.mark.parametrize("ns,nd", [(0, 0), (1, 0), (0, 1), (5, 3), (128, 0), (100, 60), (700, 333)])
def test_edwards_precomputed_matches_plain_msm(eng, oracle, ns, nd):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(1000 * ns + nd)
    static_pts = rand_points(oracle, rnd, ns)
    dyn_pts = rand_points(oracle, rnd, nd)
    if ns >= 5:
        static_pts[2] = oracle.identity(); static_pts[3] = oracle.decompress(b32(0))      # identity, order-4 point
    ss = [b32(rnd.randrange(pyref.L)) for _ in range(ns)]
    ds = [b32(rnd.randrange(pyref.L)) for _ in range(nd)]
    if ns >= 5:
        ss[0] = b32(0); ss[1] = b32(2**255 - 1); ss[4] = b32(pyref.L - 1)
    pre = pkg.VartimeEdwardsPrecomputation([oracle.compress(p) for p in static_pts], engine=eng)
    assert len(pre) == ns and pre.is_empty() == (ns == 0)
    want = oracle.compress(oracle.msm("optional", ss + ds, static_pts + dyn_pts)) if ns + nd else oracle.compress(oracle.identity())
    got = pre.vartime_mixed_multiscalar_mul(ss, ds, [oracle.compress(p) for p in dyn_pts])
    assert got == want
    if ns + nd <= 200:                                          # the reference's own algorithm (precomputed_straus.rs:57-126)
        assert oracle.compress(oracle.precomputed_straus(ss, static_pts, ds, dyn_pts)) == want
    # the object is reusable: a second call with other scalars, static part only
    ss2 = [b32(rnd.randrange(pyref.L)) for _ in range(ns)]
    want2 = oracle.compress(oracle.msm("optional", ss2, static_pts)) if ns else oracle.compress(oracle.identity())
    assert pre.vartime_multiscalar_mul(ss2) == want2
    # and agrees with the engine's non-precomputed path
    if ns + nd:
        rc, plain, _ = eng.edwards_vartime_msm(b"".join(ss + ds), b"".join(oracle.compress(p) for p in static_pts + dyn_pts), ns + nd)
        assert rc == 0 and plain == want
    pre.close()


def test_edwards_precomputed_fewer_scalars_and_errors(eng, oracle):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(77)
    static_pts = rand_points(oracle, rnd, 40)
    enc = [oracle.compress(p) for p in static_pts]
    pre = pkg.VartimeEdwardsPrecomputation(enc, engine=eng)
    # fewer static scalars than points: the unused points are ignored (traits.rs:314-316)
    ss = [b32(rnd.randrange(pyref.L)) for _ in range(17)]
    assert pre.vartime_multiscalar_mul(ss) == oracle.compress(oracle.msm("optional", ss, static_pts[:17]))
    # more static scalars than points is an error (the reference asserts)
    with pytest.raises(AssertionError):
        pre.vartime_multiscalar_mul([b32(1)] * 41)
    out = (C.c_uint8 * 32)()
    rc = eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, bytes(32 * 41), 41, None, None, 0, 0, C.addressof(out), None)
    assert rc == -1
    # optional form: an undecodable / None dynamic point gives None (traits.rs:402-413)
    dyn = rand_points(oracle, rnd, 6)
    denc = [oracle.compress(p) for p in dyn]
    ds = [b32(rnd.randrange(pyref.L)) for _ in range(6)]
    assert pre.optional_mixed_multiscalar_mul(ss, ds, denc) == oracle.compress(oracle.msm("optional", ss + ds, static_pts[:17] + dyn))
    bad = list(denc); bad[4] = b32(2)
    assert pre.optional_mixed_multiscalar_mul(ss, ds, bad) is None
    bad[4] = None
    assert pre.optional_mixed_multiscalar_mul(ss, ds, bad) is None
    with pytest.raises(ValueError):
        pre.vartime_mixed_multiscalar_mul(ss, ds, [b32(2)] * 6)
    # an undecodable static point is refused at construction
    with pytest.raises(ValueError):
        pkg.VartimeEdwardsPrecomputation(enc[:3] + [b32(2)], engine=eng)
    # extended-limb static and dynamic points (the reference's in-memory EdwardsPoint, Z != 1)
    ext = (C.c_uint64 * (20 * 40))()
    for i, p in enumerate(static_pts):
        q = oracle.sub(oracle.add(oracle.double(p), p), oracle.double(p))
        for k, v in enumerate(oracle.p3_limbs(q)):
            ext[20 * i + k] = v
    pre2 = pkg.VartimeEdwardsPrecomputation((ext, 40), engine=eng, fmt=pkg.POINTS_EXTENDED)
    ss40 = [b32(rnd.randrange(pyref.L)) for _ in range(40)]
    assert pre2.vartime_mixed_multiscalar_mul(ss40, ds, denc) == oracle.compress(oracle.msm("optional", ss40 + ds, static_pts + dyn))
    pre.close(); pre2.close()


def test_ristretto_precomputed(eng, oracle, kat):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(78)
    G = oracle.ristretto_decompress(bytes.fromhex(kat["constants"]["RISTRETTO_BASEPOINT_COMPRESSED"]["hex"]))
    ts = [rnd.randrange(pyref.L) for _ in range(90)]
    us = [rnd.randrange(pyref.L) for _ in range(50)]
    static_enc = [oracle.ristretto_compress(oracle.scalarmul(b32(t), G)) for t in ts]
    dyn_enc = [oracle.ristretto_compress(oracle.scalarmul(b32(u), G)) for u in us]
    ss = [rnd.randrange(pyref.L) for _ in range(90)]
    ds = [rnd.randrange(pyref.L) for _ in range(50)]
    pre = pkg.VartimeRistrettoPrecomputation(static_enc, engine=eng)
    total = (sum(a * t for a, t in zip(ss, ts)) + sum(a * u for a, u in zip(ds, us))) % pyref.L
    want = oracle.ristretto_compress(oracle.scalarmul(b32(total), G))
    assert pre.vartime_mixed_multiscalar_mul([b32(x) for x in ss], [b32(x) for x in ds], dyn_enc) == want
    want_s = oracle.ristretto_compress(oracle.scalarmul(b32(sum(a * t for a, t in zip(ss, ts)) % pyref.L), G))
    assert pre.vartime_multiscalar_mul([b32(x) for x in ss]) == want_s
    # i*G for the reference's 16 small multiples (C/ristretto.rs:1387-1461): static = [G], scalar = i
    encs = [bytes.fromhex(h) for h in kat["ristretto"]["SMALL_MULTIPLES"]["hex"]]
    preG = pkg.VartimeRistrettoPrecomputation([encs[1]], engine=eng)
    assert [preG.vartime_multiscalar_mul([b32(i)]) for i in range(16)] == encs
    # a negative-s encoding is not a Ristretto point: None / refused
    assert pre.optional_mixed_multiscalar_mul([], [b32(1)], [b32(1)]) is None
    with pytest.raises(ValueError):
        pkg.VartimeRistrettoPrecomputation([b32(1)], engine=eng)
    pre.close(); preG.close()


def test_precomputed_large_reuse(eng, oracle):
    """2^17 static generators t_j*B made on the GPU, resident once; three calls with fresh scalars checked through
    sum b_j (t_j B) = (sum b_j t_j) B (the identity of C/edwards.rs:2276-2335)."""
    import numpy as np
    import curve25519_dalek_b200 as pkg
    n = 1 << 17
    rng = np.random.Generator(np.random.PCG64(11))
    t = rng.integers(0, 256, size=(n, 32), dtype=np.uint8); t[:, 31] &= 0x0F
    limbs, _ = eng.mul_base_batch(t, n, want_compressed=False)
    pre = pkg.VartimeEdwardsPrecomputation((limbs, n), engine=eng, fmt=pkg.POINTS_EXTENDED)
    tv = [int.from_bytes(t[i].tobytes(), "little") for i in range(n)]
    B = oracle.basepoint()
    for trial in range(3):
        s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8); s[:, 31] &= 0x0F
        out = (C.c_uint8 * 32)()
        rc = eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, s.ctypes.data, n, None, None, 1, 0, C.addressof(out), None)
        assert rc == 0
        total = sum(int.from_bytes(s[i].tobytes(), "little") * tv[i] for i in range(n)) % pyref.L
        assert bytes(out) == oracle.compress(oracle.scalarmul(b32(total), B))
    pre.close()


@pytest.mark.parametrize("tables", [1, 0])
def test_precomputed_window_tables(eng, oracle, tables):
    """>= 4096 static points keep the tables 2^(c w) P_i (one bucket window, no doublings).  With and without them:
    full and partial static scalar lists, dynamic points of their own width, edge scalars, all against
    sum b_j (t_j B) + sum a_i (u_i B) = (sum b_j t_j + sum a_i u_i) B computed by the oracle."""
    import numpy as np
    import curve25519_dalek_b200 as pkg
    n, nd = 5000, 37
    rng = np.random.Generator(np.random.PCG64(21))
    t = rng.integers(0, 256, size=(n, 32), dtype=np.uint8); t[:, 31] &= 0x0F
    t[7] = 0; t[8] = 0; t[8, 0] = 1                                  # identity and B itself among the static points
    u = rng.integers(0, 256, size=(nd, 32), dtype=np.uint8); u[:, 31] &= 0x0F
    limbs, _ = eng.mul_base_batch(t, n, want_compressed=False)
    dlimbs, dcomp = eng.mul_base_batch(u, nd)
    tv = [int.from_bytes(t[i].tobytes(), "little") for i in range(n)]
    uv = [int.from_bytes(u[i].tobytes(), "little") for i in range(nd)]
    B = oracle.basepoint()
    found = eng.get_option("precomp_tables")
    eng.set_option("precomp_tables", tables)
    try:
        pre = pkg.VartimeEdwardsPrecomputation((limbs, n), engine=eng, fmt=pkg.POINTS_EXTENDED)
    finally:
        eng.set_option("precomp_tables", found)
    for ns in (n, 4097, 1):
        b = rng.integers(0, 256, size=(ns, 32), dtype=np.uint8); b[:, 31] &= 0x1F
        b[0] = 255; b[0, 31] = 0x7F                                   # 2^255 - 1
        if ns > 3:
            b[1] = 0; b[2] = 0; b[2, 0] = 1
        a = rng.integers(0, 256, size=(nd, 32), dtype=np.uint8); a[:, 31] &= 0x0F
        bv = [int.from_bytes(b[i].tobytes(), "little") for i in range(ns)]
        av = [int.from_bytes(a[i].tobytes(), "little") for i in range(nd)]
        for dyn in (False, True):
            total = sum(x * y for x, y in zip(bv, tv)) + (sum(x * y for x, y in zip(av, uv)) if dyn else 0)
            want = oracle.compress(oracle.scalarmul(b32(total % pyref.L), B))
            out = (C.c_uint8 * 32)()
            rc = eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, b.ctypes.data, ns, a.ctypes.data if dyn else None,
                                                      C.cast(dlimbs, C.c_void_p).value if dyn else None, 1, nd if dyn else 0,
                                                      C.addressof(out), None)
            assert rc == 0 and bytes(out) == want, (tables, ns, dyn)
    # compressed dynamic points, one of them undecodable -> None
    enc = bytearray(dcomp); enc[32 * 5:32 * 6] = b32(2)
    out = (C.c_uint8 * 32)()
    a = rng.integers(0, 256, size=(nd, 32), dtype=np.uint8); a[:, 31] &= 0x0F
    b = rng.integers(0, 256, size=(n, 32), dtype=np.uint8); b[:, 31] &= 0x0F
    ebuf = (C.c_uint8 * len(enc)).from_buffer(enc)
    assert eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, b.ctypes.data, n, a.ctypes.data, C.addressof(ebuf), 0, nd, C.addressof(out), None) == 1
    pre.close()
