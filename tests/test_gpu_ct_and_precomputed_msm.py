"""GPU tests of the constant-time MSM and of the precomputed MSM on the code paths of their own.

MultiscalarMul::multiscalar_mul (dalek_b200_edwards_ct_msm, csrc/straus.cu): k_ct_scalar_mul computes s_i P_i, one
thread per term in 64-thread blocks, and k_sum_level sums the products in a tree of fan-in 8 (64 outputs, so 512 inputs,
per block).  The sizes reach tree depths 0 to 7, levels whose last group holds a single point (8^k + 1) or whose input is
exactly 8^k, and the block edges of both kernels.  The contract is s P for any scalar below 2^255 on any point: the
scalar is not reduced mod l, so on a point with a torsion component s and s mod l give different results.

VartimePrecomputedMultiscalarMul (csrc/precomp.cu): 2^18 or more static scalars are copied and accumulated in
K = min(4, host_chunks) chunks, each chunk folding into the buckets of the earlier ones; with window tables every chunk
reads its own slice of each table (the tables have a stride of n points).  Ristretto precomputations with tables add the
dynamic part's result to the static part's before the Ristretto encoding; the dynamic part picks its own window width
at every call, on either side of the tables' width.  Then the argument rules of a call.

Expected values: msm_pool's exact identity for any scalar below 2^256 and any E[8] component, and the oracle's
multiscalar_mul (a Straus restatement) where it is fast enough."""
import contextlib
import ctypes as C
import random
import types

import numpy as np
import pytest

import msm_digit_cases as mdc
import msm_pool
import point_checks
from msm_pool import L, b32, scalar_array, scalar_ints
from test_gpu_ristretto import cosets  # noqa: F401  (fixture: the identity and 64 points t B, each as P + T, T in E[4], Z != 1)

pytestmark = pytest.mark.gpu
OPTIONS = ("precomp_tables", "host_chunks", "window_bits")
E_INVALID_ARG = -1


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    found = {k: e.get_option(k) for k in OPTIONS}
    yield e
    assert {k: e.get_option(k) for k in OPTIONS} == found          # no test leaves an option changed
    e.close()


@contextlib.contextmanager
def options(eng, **opts):
    """the options for the body of the block; each is restored to the value it had before"""
    found = {k: eng.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            eng.set_option(k, v)
        yield
    finally:
        for k, v in found.items():
            eng.set_option(k, v)


@pytest.fixture(scope="module")
def pool(oracle):
    return msm_pool.Pool(oracle)


def width_of(eng, n):
    """the window width the engine picks for n pairs (the window count 256 // c + 1 tells c = 4 .. 20 apart)"""
    nwin = eng.msm_window_count(n)
    (c,) = [c for c in range(4, 21) if mdc.window_count(c) == nwin]
    return c


def place(arr, start, rows):
    """arr[start + k] = rows[k] for the k that fall inside arr"""
    for k, r in enumerate(rows):
        if 0 <= start + k < len(arr):
            arr[start + k] = r


# ---- 1. constant-time MSM ----
ALL8 = int("8" * 63, 16)        # radix-16 digits -8, -7, ..., -7, 1: a carry through all 63 digits
CT_EDGES = [0, 1, L - 1, L, L + 1, 2**252, 2**255 - 1, ALL8, (7 << 252) + ALL8, int("7" * 64, 16)]   # top digits 8, 8; all-7: no carry
CT_SIZES = [1, 7, 8, 9, 63, 64, 65, 511, 512, 513, 4095, 4096, 4097, 32768, 32769, 2**17 + 3, 2**18 + 1]
CT_EDGES_AT = (8, 64, 512, 4096, 32768, 2**18)      # group and block edges of both kernels
ORACLE_MAX = 513


@pytest.fixture(scope="module")
def ct_cases(pool):
    cache = {}

    def case(n):
        """(scalars (n, 32) uint8, pool indices, expected encoding).  Even scalars below 2^252, odd ones in [2^253, 2^255);
        the edge scalars around each edge and at the first and last indices; the points of E[8] (the identity among them)
        at the first indices, just below each edge and just below the last edge scalars; about one point in eight
        shifted by T8.  The last term is the all-7 scalar on a point with a prime-order part, so that the product a
        level's lone last group holds (n = 8^k + 1) is never the identity."""
        if n not in cache:
            rng = np.random.Generator(np.random.PCG64(n))
            s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
            s[0::2, 31] &= 0x0F
            s[1::2, 31] = (s[1::2, 31] & 0x7F) | 0x20
            idx = pool.random_indices(rng, n)
            edges, e = scalar_array(CT_EDGES), len(CT_EDGES)
            tors = msm_pool.E8 + np.arange(8)
            for st in [b - e // 2 for b in CT_EDGES_AT if b < n] + [0, n - e]:
                place(s, st, edges)
            for st in [b - 8 for b in CT_EDGES_AT if b < n] + [0, n - e - 8]:
                place(idx, st, tors)
            idx[-1] = 0
            assert not (s[:, 31] & 0x80).any()
            cache[n] = (s, idx, pool.want(scalar_ints(s), idx))
        return cache[n]

    return case


@pytest.mark.parametrize("n", CT_SIZES)
def test_ct_msm_sizes(eng, oracle, pool, ct_cases, n):
    s, idx, want = ct_cases(n)
    comp = pool.comp[idx]
    rc, got, limbs = eng.edwards_ct_msm(s, comp, n, want_limbs=True)
    assert rc == 0 and got == want
    point_checks.check_limbs(limbs, want, what="compressed input")
    ext = pool.extended(idx, random.Random(n))
    rc, got_ext, limbs = eng.edwards_ct_msm(s, ext, n, point_fmt=1, want_limbs=True)
    assert rc == 0 and got_ext == want
    point_checks.check_limbs(limbs, want, what="extended input")
    rc, got_vt, _ = eng.edwards_vartime_msm(s, comp, n)
    assert rc == 0 and got_vt == want
    if n <= ORACLE_MAX:
        pts = [pool.points[j] for j in idx.tolist()]
        assert oracle.compress(oracle.msm_ct([bytes(r) for r in s], pts)) == want


def test_ct_msm_rejects_bit_255_before_any_launch(eng, pool, ct_cases):
    import curve25519_dalek_b200 as pkg
    n = 2**17 + 3
    s, idx, want = ct_cases(n)
    comp = pool.comp[idx]
    bad = s.copy()
    bad[-1, 31] |= 0x80                                            # the last scalar only
    l0 = eng.launch_count()
    with pytest.raises(pkg.EngineError, match="bit 255"):
        eng.edwards_ct_msm(bad, comp, n)
    assert eng.launch_count() == l0
    rc, got, _ = eng.edwards_ct_msm(s, comp, n)
    assert rc == 0 and got == want


def test_ct_msm_undecodable_point_and_empty_input(eng, oracle, pool, ct_cases):
    import curve25519_dalek_b200 as pkg
    n = 4097
    s, idx, want = ct_cases(n)
    assert oracle.decompress(b32(2)) is None
    comp = pool.comp[idx].copy()
    comp[-1] = np.frombuffer(b32(2), dtype=np.uint8)
    with pytest.raises(pkg.EngineError):
        eng.edwards_ct_msm(s, comp, n)
    assert "does not decode" in eng.lib.dalek_b200_last_error(eng.h).decode()
    rc, got, _ = eng.edwards_ct_msm(s, pool.comp[idx], n)
    assert rc == 0 and got == want
    rc, got, limbs = eng.edwards_ct_msm(b"", b"", 0, want_limbs=True)
    assert rc == 0 and got == b32(1)
    point_checks.check_limbs(limbs, b32(1))


def test_edwards_python_msm_wrappers(eng, pool, ct_cases):
    import curve25519_dalek_b200 as pkg
    E = pkg.EdwardsPoint
    s, idx, want = ct_cases(65)
    ss = [bytes(r) for r in s]
    pts = [bytes(r) for r in pool.comp[idx]]
    assert E.multiscalar_mul(ss, pts, engine=eng) == want
    assert E.optional_multiscalar_mul(ss, pts, engine=eng) == want
    assert E.vartime_multiscalar_mul(ss, pts, engine=eng) == want
    for bad in (None, b32(2)):
        pb = pts[:-1] + [bad]
        assert E.optional_multiscalar_mul(ss, pb, engine=eng) is None
        with pytest.raises(ValueError):
            E.vartime_multiscalar_mul(ss, pb, engine=eng)
    with pytest.raises(pkg.EngineError):                           # multiscalar_mul takes points, not Options
        E.multiscalar_mul(ss, pts[:-1] + [b32(2)], engine=eng)
    for f in (E.multiscalar_mul, E.optional_multiscalar_mul, E.vartime_multiscalar_mul):
        with pytest.raises(AssertionError):
            f(ss, pts[:-1], engine=eng)
    assert E.vartime_multiscalar_mul(ss, pts, engine=eng) == want


# ---- 2. precomputed MSM ----
def precomp_msm(eng, pre, ss, ns, ds=None, dp=None, fmt=0, nd=0):
    """(rc, out) of dalek_b200_precomp_mixed_msm on host arrays; rc is returned, not raised"""
    out = (C.c_uint8 * 32)()
    rc = eng.lib.dalek_b200_precomp_mixed_msm(eng.h, pre.h, ss.ctypes.data if ns else None, ns,
                                              ds.ctypes.data if nd else None, dp.ctypes.data if nd else None, fmt, nd,
                                              C.addressof(out), None)
    return rc, bytes(out)


def build_pair(eng, cls, points):
    """{1: the precomputation with window tables, 0: without}; the tables were built (k_precomp_table, one launch)"""
    pres, launches = {}, {}
    for tables in (1, 0):
        with options(eng, precomp_tables=tables):
            l0 = eng.launch_count()
            pres[tables] = cls(points, engine=eng)
            launches[tables] = eng.launch_count() - l0
    assert launches[1] == launches[0] + 1
    return pres


def close_all(pres):
    for p in pres.values():
        p.close()


N_CHUNKED = 2**18 + 5
STATIC_COUNTS = (N_CHUNKED, 2**18, 2**18 - 1)      # K > 1 on the whole list and on exactly 2^18; K = 1 just below
N_DYN = 37


@pytest.fixture(scope="module")
def chunked(eng, pool):
    """N_CHUNKED compressed pool points with and without tables; full-width static scalars with 2^256 - 1 and the
    boundary scalars of the tables' width on both sides of every chunk boundary; N_DYN dynamic terms"""
    import curve25519_dalek_b200 as pkg
    ch = types.SimpleNamespace()
    n = N_CHUNKED
    rng = np.random.Generator(np.random.PCG64(218))
    idx = pool.random_indices(rng, n)
    place(idx, 100, msm_pool.E8 + np.arange(8))
    ch.pres = build_pair(eng, pkg.VartimeEdwardsPrecomputation, [bytes(r) for r in pool.comp[idx]])
    ch.c = width_of(eng, n)
    ss = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    edges = scalar_array([2**256 - 1] + mdc.boundary_scalars(ch.c))
    e = len(edges)
    place(ss, 0, edges)
    place(ss, n - e, edges)
    for ns in STATIC_COUNTS[:2]:
        for K in (2, 3, 4):
            for k in range(1, K):
                place(ss, ns * k // K - e // 2, edges)
    ints = scalar_ints(ss)
    ch.ss = ss
    ch.static_sums = {ns: pool.sums(ints[:ns], idx[:ns]) for ns in STATIC_COUNTS}
    ch.ds = rng.integers(0, 256, size=(N_DYN, 32), dtype=np.uint8)
    ch.ds[0] = 255
    didx = pool.random_indices(rng, N_DYN)
    place(didx, 1, msm_pool.E8 + np.arange(8))
    ch.dyn = {0: pool.comp[didx].copy(), 1: pool.extended(didx, random.Random(N_DYN))}
    ch.dyn_sums = pool.sums(scalar_ints(ch.ds), didx)
    yield ch
    close_all(ch.pres)


@pytest.mark.parametrize("host_chunks", [1, 2, 3, 4, 8])
def test_precomputed_chunked_static_scalars(eng, pool, chunked, host_chunks):
    """host_chunks 1, 2, 3, 4, 8: K = 1, 2, 3, 4, 4 chunks at 2^18 static scalars and more"""
    ch = chunked
    fmt = host_chunks % 2                           # extended dynamic points with 1 and 3 chunks, compressed otherwise
    with options(eng, host_chunks=host_chunks):
        for ns in STATIC_COUNTS:
            for dyn in (False, True):
                k, m = ch.static_sums[ns]
                if dyn:
                    k, m = k + ch.dyn_sums[0], m + ch.dyn_sums[1]
                want = (0, pool.encode(k, m))
                nd = N_DYN if dyn else 0
                for tables in (1, 0):
                    assert precomp_msm(eng, ch.pres[tables], ch.ss, ns, ch.ds, ch.dyn[fmt], fmt, nd) == want, (ns, dyn, tables)


def ristretto_encode(oracle, pool, k):
    return oracle.ristretto_compress(oracle.scalarmul(b32(k % L), pool.B))


@pytest.mark.parametrize("n", [4097, N_CHUNKED])
def test_ristretto_precomputed_tables(eng, oracle, pool, cosets, n):
    """static Ristretto encodings with and without tables; dynamic terms as Ristretto encodings, or as extended limbs
    of P + T for each T in E[4] (rescaled): the Ristretto sum, whichever representatives the dynamic points are"""
    import curve25519_dalek_b200 as pkg
    rng = np.random.Generator(np.random.PCG64(n))
    ts = [t for _, t, _ in cosets]
    encs = np.frombuffer(b"".join(oracle.ristretto_compress(P) for P, _, _ in cosets), dtype=np.uint8).reshape(-1, 32)
    sidx = rng.integers(0, len(cosets), size=n)
    ss = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    place(ss, 0, scalar_array(mdc.EDGE_SCALARS))
    k_static = sum(s * ts[j] for s, j in zip(scalar_ints(ss), sidx.tolist()))
    nd = 41
    didx = rng.integers(0, len(cosets), size=nd)
    ds = rng.integers(0, 256, size=(nd, 32), dtype=np.uint8)
    k_dyn = sum(s * ts[j] for s, j in zip(scalar_ints(ds), didx.tolist()))
    r_dyn = encs[didx].copy()
    want_s, want = ristretto_encode(oracle, pool, k_static), ristretto_encode(oracle, pool, k_static + k_dyn)
    pres = build_pair(eng, pkg.VartimeRistrettoPrecomputation, [bytes(r) for r in encs[sidx]])
    try:
        for tables, pre in pres.items():
            assert precomp_msm(eng, pre, ss, n) == (0, want_s), tables
            assert precomp_msm(eng, pre, ss, n, ds, r_dyn, 2, nd) == (0, want), tables
            for t in range(4):                      # every dynamic point P + T for the same T, then mixed T
                ext = np.array([cosets[j][2][t] for j in didx.tolist()], dtype=np.uint64)
                assert precomp_msm(eng, pre, ss, n, ds, ext, 1, nd) == (0, want), (tables, t)
            ext = np.array([cosets[j][2][i % 4] for i, j in enumerate(didx.tolist())], dtype=np.uint64)
            assert precomp_msm(eng, pre, ss, n, ds, ext, 1, nd) == (0, want), tables
    finally:
        close_all(pres)


def test_precomputed_tables_dynamic_widths(eng, pool):
    """tables at the width of 4097 points; the dynamic part picks its own width from its count, on both sides of the
    tables' width, or takes window_bits when it is set after construction; the static part keeps the tables' width"""
    import curve25519_dalek_b200 as pkg
    n = 4097
    rng = np.random.Generator(np.random.PCG64(4097))
    idx = pool.random_indices(rng, n)
    pres = build_pair(eng, pkg.VartimeEdwardsPrecomputation, [bytes(r) for r in pool.comp[idx]])
    try:
        c = width_of(eng, n)
        counts = (1, 189, 190, 2**16 + 1)
        widths = [width_of(eng, nd) for nd in counts]
        assert min(widths) < c < max(widths), (c, widths)
        ss = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        place(ss, 0, scalar_array(mdc.boundary_scalars(c)))
        k0, m0 = pool.sums(scalar_ints(ss), idx)
        for nd in counts:
            ds = rng.integers(0, 256, size=(nd, 32), dtype=np.uint8)
            place(ds, 0, scalar_array(mdc.boundary_scalars(width_of(eng, nd))))
            didx = pool.random_indices(rng, nd)
            k, m = pool.sums(scalar_ints(ds), didx)
            want = (0, pool.encode(k0 + k, m0 + m))
            dp = pool.comp[didx].copy()
            for wb in (0, 4, 20):
                with options(eng, window_bits=wb):
                    for tables, pre in pres.items():
                        assert precomp_msm(eng, pre, ss, n, ds, dp, 0, nd) == want, (nd, wb, tables)
    finally:
        close_all(pres)


def test_precomputed_argument_rules(eng, oracle, pool, cosets):
    """each call is refused with DALEK_E_INVALID_ARG before any launch, and the next valid call is correct"""
    import curve25519_dalek_b200 as pkg
    rng = np.random.Generator(np.random.PCG64(31))
    n = 9
    idx = pool.random_indices(rng, n)
    ed = pkg.VartimeEdwardsPrecomputation([bytes(r) for r in pool.comp[idx]], engine=eng)
    renc = np.frombuffer(b"".join(oracle.ristretto_compress(P) for P, _, _ in cosets[:n]), dtype=np.uint8).reshape(n, 32)
    ri = pkg.VartimeRistrettoPrecomputation([bytes(r) for r in renc], engine=eng)
    other = pkg.Engine(0)
    try:
        ss = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        ds = rng.integers(0, 256, size=(3, 32), dtype=np.uint8)
        ints = scalar_ints(ss)
        ed_want = (0, pool.want(ints, idx))
        ri_want = (0, ristretto_encode(oracle, pool, sum(s * cosets[j][1] for j, s in enumerate(ints))))
        r_dyn, e_dyn = renc[:3].copy(), pool.comp[:3].copy()
        refused = [
            ("Edwards precomputation, Ristretto dynamic points", eng, ed, dict(ds=ds, dp=r_dyn, fmt=2, nd=3)),
            ("Ristretto precomputation, compressed Edwards dynamic points", eng, ri, dict(ds=ds, dp=e_dyn, fmt=0, nd=3)),
            ("another context", other, ed, {}),
            ("another context", other, ri, {}),
            # the buffers hold 9 and 3 entries: the call must not read them
            ("n_static + n_dynamic = 2^31", eng, ed, dict(ds=ds, dp=e_dyn, fmt=0, nd=2**31 - n)),
        ]
        for what, e, pre, kw in refused:
            l0 = e.launch_count()
            assert precomp_msm(e, pre, ss, n, **kw)[0] == E_INVALID_ARG, what
            assert e.launch_count() == l0, what
            assert precomp_msm(eng, ed, ss, n) == ed_want, what
            assert precomp_msm(eng, ri, ss, n) == ri_want, what
    finally:
        ed.close()
        ri.close()
        other.close()


# ---- 3. Python wrapper of the Ristretto double-base batch ----
def test_ristretto_double_base_batch_wrapper(eng, kat):
    import curve25519_dalek_b200 as pkg
    encs = [bytes.fromhex(h) for h in kat["ristretto"]["SMALL_MULTIPLES"]["hex"]]
    ints = b"".join(b32(i) for i in range(16))
    zeros = bytes(32 * 16)
    G, H = encs[1], encs[3]
    for a, b, mult in ((ints, zeros, 1), (zeros, ints, 3)):       # i G, then i H = 3i G
        got = pkg.RistrettoPoint.double_base_batch(a, b, G, H, engine=eng)
        rc, raw = eng.ristretto_double_base_batch(a, b, G, H, 16)
        assert rc == 0 and got == raw
        assert [got[32 * i:32 * i + 32] for i in range(16) if mult * i < 16] == [encs[mult * i] for i in range(16) if mult * i < 16]
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.double_base_batch(ints, zeros, b32(1), H, engine=eng)
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.double_base_batch(ints, zeros, G, b32(1), engine=eng)
