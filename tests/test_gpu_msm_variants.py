"""GPU tests of the bucket MSM under every compilation of its bucket kernel, at every window width, on the scalars
whose signed digits reach the edges of k_digits (tests/msm_digit_cases.py).

The options field_f64 and acc_tma select one of three forms of k_bucket_accumulate (csrc/msm.cu): <1,0> on the FP64-pipe
field with cp.async gathers (the default), <1,1> on the same field with TMA bulk copies completing on mbarriers, and
<0,0> on the IMAD.WIDE field.  field_f64 = 0 also runs level 0 of the bucket reduction in k_chunk_reduce (one_based = 1),
sends MSMs below 190 pairs to the bucket pipeline instead of vartime Straus, and turns off the per-key comb of
verify_each.  No option may change a result.

Every reference is exact and cheap: the points are t_j B from a pool of oracle points, some of them shifted by the
order-8 point T8, so that sum s_i P_i = ((sum s_i t_i) mod l) B + ((sum of the s_i of shifted points) mod 8) T8."""
import contextlib
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import msm_digit_cases as mdc
import pyref
import torsion_cases
from test_gpu_msm_affine_prep import coords, limbs_of
from test_gpu_verify_each import flat as flat_msgs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L

NPOOL, NTORS = 64, 8             # pool entries NPOOL + k are entry k shifted by T8
VARIANTS = {"f64": (1, 0), "f64_tma": (1, 1), "imad": (0, 0)}     # name: (field_f64, acc_tma)
DEFAULTS = dict(field_f64=1, acc_tma=0, window_bits=0, host_chunks=8, precomp_tables=0, each_comb=1)
N_BOUNDARY = 2000                # pairs per boundary-digit case: the boundary scalars plus seeded filler


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@contextlib.contextmanager
def options(eng, variant="f64", **opts):
    """the bucket-kernel variant and further options for the body of the block; all of them are reset afterwards"""
    f64, tma = VARIANTS[variant]
    opts = dict(field_f64=f64, acc_tma=tma, **opts)
    try:
        for k, v in opts.items():
            eng.set_option(k, v)
        yield
    finally:
        for k in opts:
            eng.set_option(k, DEFAULTS[k])


def b32(x):
    return x.to_bytes(32, "little")


def rescaled_limbs(xyzt, rnd):
    """the extended point (X : Y : Z : T) as (lambda X : lambda Y : lambda Z : lambda T), lambda != 0, 1 drawn from rnd"""
    lam = rnd.randrange(2, pyref.p)
    return limbs_of([v * lam % pyref.p for v in xyzt])


def width_of(eng, n):
    """the window width the engine picks for n pairs (the window count 256 // c + 1 tells c = 4 .. 20 apart)"""
    nwin = eng.msm_window_count(n)
    (c,) = [c for c in range(4, 21) if mdc.window_count(c) == nwin]
    return c


class Pool:
    def __init__(self, oracle):
        self.oracle = oracle
        rnd = random.Random(0xB0C4E7)
        self.B = oracle.basepoint()
        self.T8 = oracle.decompress(torsion_cases.T8)
        self.t = [rnd.randrange(1, L) for _ in range(NPOOL)]
        pts = [oracle.scalarmul(b32(t), self.B) for t in self.t]
        self.points = pts + [oracle.add(p, self.T8) for p in pts[:NTORS]]
        self.comp = [oracle.compress(p) for p in self.points]
        self.xyzt = [coords(oracle.p3_limbs(p)) for p in self.points]
        self.cases = {}

    def want(self, scalars, idx):
        k = sum(s * self.t[j % NPOOL] for s, j in zip(scalars, idx)) % L
        m = sum(s for s, j in zip(scalars, idx) if j >= NPOOL) % 8
        r = self.oracle.scalarmul(b32(k), self.B)
        if m:
            r = self.oracle.add(r, self.oracle.scalarmul(b32(m), self.T8))
        return self.oracle.compress(r)

    def inputs(self, scalars, idx, rnd):
        """(scalars, compressed points, extended points with every point rescaled by its own lambda != 1)"""
        sb = b"".join(b32(s) for s in scalars)
        comp = b"".join(self.comp[j] for j in idx)
        ext = np.empty((len(idx), 20), dtype=np.uint64)
        for i, j in enumerate(idx):
            ext[i] = rescaled_limbs(self.xyzt[j], rnd)
        return sb, comp, ext

    def boundary_case(self, c, n=N_BOUNDARY, seed=0):
        """boundary_scalars(c) and seeded filler (half of it above l, up to 2^256 - 1) on pool points, one in 37
        shifted by T8: (scalars, compressed, extended, want)"""
        key = (c, n, seed)
        if key not in self.cases:
            rnd = random.Random(1000 * seed + c)
            scalars = mdc.boundary_scalars(c)
            scalars = scalars + [rnd.getrandbits(256) if k % 2 else rnd.randrange(L) for k in range(n - len(scalars))]
            idx = [NPOOL + rnd.randrange(NTORS) if i % 37 == 5 else rnd.randrange(NPOOL) for i in range(n)]
            self.cases[key] = self.inputs(scalars, idx, rnd) + (self.want(scalars, idx),)
        return self.cases[key]


@pytest.fixture(scope="module")
def pool(oracle):
    return Pool(oracle)


def check_msm(eng, oracle, want, *args, **kw):
    rc, got, limbs = eng.edwards_vartime_msm(*args, want_limbs=True, **kw)
    assert rc == 0 and got == want
    assert oracle.compress(oracle.p3_from_limbs(limbs)) == want         # the returned limbs are the same point


# ---- a. boundary digits at every width, on every kernel form ----
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("c", range(4, 21))
def test_boundary_digits_every_width(eng, oracle, pool, c, variant):
    """c = 17 .. 20: 2^16 .. 2^19 buckets per window and up to six reduction levels; c = 20 takes k_scan_bases to its
    128 parts and cuts each 32768-entry W array of k_plain_sum into 128 pieces."""
    import torch
    sb, comp, ext, want = pool.boundary_case(c)
    n = N_BOUNDARY
    dev = torch.device("cuda", 0)
    d_s = torch.frombuffer(bytearray(sb), dtype=torch.uint8).to(dev)
    d_p = torch.from_numpy(ext.view(np.int64)).to(dev)
    torch.cuda.synchronize()
    with options(eng, variant, window_bits=c):
        assert eng.msm_window_count(n) == mdc.window_count(c)
        check_msm(eng, oracle, want, sb, comp, n, point_fmt=0)
        check_msm(eng, oracle, want, sb, ext, n, point_fmt=1)
        check_msm(eng, oracle, want, d_s.data_ptr(), d_p.data_ptr(), n, point_fmt=1, device_ptrs=True)


# ---- b. buckets cut into tasks: k_heavy_fixup on the task sums of each kernel form ----
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_heavy_buckets(eng, oracle, pool, variant):
    rnd = random.Random(700)
    n = 700
    c = width_of(eng, n)
    idx = [rnd.randrange(NPOOL + NTORS) for _ in range(n)]
    _, comp, _ = pool.inputs([], idx, rnd)
    # every point in one bucket of each window: the last bucket of every full window, then arbitrary buckets
    for s in (mdc.boundary_scalars(c)[0], rnd.getrandbits(256)):
        with options(eng, variant):
            rc, got, _ = eng.edwards_vartime_msm(b32(s) * n, comp, n)
        assert rc == 0 and got == pool.want([s] * n, idx), hex(s)
    # c = 17: a third of the scalars equal, -(2^16 - 1) with a carry in every full window
    n, c = N_BOUNDARY, 17
    scalars = mdc.boundary_scalars(c)
    scalars = scalars + [rnd.getrandbits(256) for _ in range(n - len(scalars))]
    heavy = mdc.boundary_scalars(c)[5]
    for i in range(0, n, 3):
        scalars[i] = heavy
    idx = [rnd.randrange(NPOOL + NTORS) for _ in range(n)]
    sb, comp, ext = pool.inputs(scalars, idx, rnd)
    want = pool.want(scalars, idx)
    with options(eng, variant, window_bits=c):
        check_msm(eng, oracle, want, sb, comp, n, point_fmt=0)
        check_msm(eng, oracle, want, sb, ext, n, point_fmt=1)


# ---- c. host buffers streamed in chunks: later chunks fold the stored bucket sums in (fold_old) ----
@pytest.fixture(scope="module")
def streamed(eng, pool):
    n = (1 << 18) + 5
    rnd = random.Random(218)
    scalars = [rnd.getrandbits(256) for _ in range(n)]
    for i in range(0, n, 3):
        scalars[i] = scalars[0]                     # heavy buckets in every chunk
    cases = mdc.boundary_scalars(width_of(eng, n))
    scalars[1:3 * len(cases):3] = cases
    idx = np.array([rnd.randrange(NPOOL + NTORS) for _ in range(n)])
    sb = np.frombuffer(b"".join(b32(s) for s in scalars), dtype=np.uint8).copy()
    comp = np.frombuffer(b"".join(pool.comp), dtype=np.uint8).reshape(-1, 32)[idx].copy()
    lim = np.array([rescaled_limbs(xyzt, rnd) for xyzt in pool.xyzt], dtype=np.uint64)
    ext = lim[idx].copy()                           # every pool entry with its own lambda
    return n, sb, comp, ext, pool.want(scalars, idx.tolist())


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_host_streamed_chunks(eng, streamed, variant):
    n, sb, comp, ext, want = streamed
    with options(eng, variant, host_chunks=3):
        for fmt, pts in ((0, comp), (1, ext)):
            for chunks in (3, 1):
                eng.set_option("host_chunks", chunks)
                rc, got, _ = eng.edwards_vartime_msm(sb, pts, n, point_fmt=fmt)
                assert rc == 0 and got == want, (fmt, chunks)


# ---- d. small MSMs with field_f64 = 0: the bucket pipeline instead of vartime Straus ----
def exact_msm(oracle, scalars, points):
    """sum s_i P_i for any 256-bit s_i and any points, s_i split as lo + 2^252 hi to stay inside the oracle's Scalar"""
    acc = oracle.identity()
    for s, p in zip(scalars, points):
        lo = oracle.scalarmul(b32(s % 2**252), p)
        hi = oracle.mul_by_pow_2(oracle.scalarmul(b32(s >> 252), p), 252)
        acc = oracle.add(acc, oracle.add(lo, hi))
    return oracle.compress(acc)


@pytest.mark.parametrize("n", [1, 2, 9, 189, 190])
def test_small_msm_imad_bucket_path(eng, oracle, pool, n):
    rnd = random.Random(n)
    scalars = [rnd.getrandbits(256) for _ in range(n)]
    edges = [2**256 - 1, 2**255, 2**255 + rnd.randrange(2**255), L, L - 1, 0, 1]
    scalars[:len(edges)] = edges[:n]
    points = [pool.points[rnd.randrange(NPOOL + NTORS)] for _ in range(n)]
    if n >= 9:
        points[6] = oracle.identity()
        points[7] = oracle.decompress(b32(0))                  # order 4
        points[8] = oracle.decompress(b32(pyref.p - 1))        # order 2
    want = exact_msm(oracle, scalars, points)
    sb = b"".join(b32(s) for s in scalars)
    comp = b"".join(oracle.compress(p) for p in points)
    ext = np.array([rescaled_limbs(coords(oracle.p3_limbs(p)), rnd) for p in points], dtype=np.uint64)
    with options(eng, "imad"):
        for fmt, pts in ((0, comp), (1, ext)):
            l0 = eng.launch_count()
            check_msm(eng, oracle, want, sb, pts, n, point_fmt=fmt)
            assert eng.launch_count() - l0 > 5, fmt           # the bucket pipeline, not the 4-launch Straus path


# ---- e. precomputed 2^(cw) P tables: every digit into one bucket window (flat mode) ----
@pytest.fixture(scope="module")
def flat_pre(eng, oracle, pool):
    import curve25519_dalek_b200 as pkg
    n = 4097
    c = width_of(eng, n)                             # the tables are built for the width of an MSM of n pairs
    rnd = random.Random(4097)
    idx = [rnd.randrange(NPOOL + NTORS) for _ in range(n)]
    enc = [pool.comp[j] for j in idx]
    launches = []
    for tables in (0, 1):
        with options(eng, precomp_tables=tables):
            l0 = eng.launch_count()
            pre = pkg.VartimeEdwardsPrecomputation(enc, engine=eng)
            launches.append(eng.launch_count() - l0)
        if not tables:
            pre.close()
    assert launches[1] == launches[0] + 1            # the tables were built (k_precomp_table)
    yield pre, idx, c
    pre.close()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_precomputed_tables_flat_mode(eng, pool, flat_pre, variant):
    pre, idx, c = flat_pre
    rnd = random.Random(41)
    ss = mdc.boundary_scalars(c)
    ss = ss + [rnd.getrandbits(256) for _ in range(len(idx) - len(ss))]
    ds = mdc.boundary_scalars(width_of(eng, 300))
    ds = ds + [rnd.getrandbits(256) for _ in range(300 - len(ds))]
    didx = [rnd.randrange(NPOOL + NTORS) for _ in range(len(ds))]
    with options(eng, variant):
        assert pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [], []) == pool.want(ss, idx)
        got = pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [b32(s) for s in ds], [pool.comp[j] for j in didx])
        assert got == pool.want(ss + ds, idx + didx)


# ---- f. sharded records at wide windows (window_bits sets the shard's width too) ----
@pytest.mark.parametrize("variant", ["f64", "imad"])
@pytest.mark.parametrize("c", [17, 20])
def test_sharded_records_wide_windows(eng, oracle, pool, c, variant):
    from curve25519_dalek_b200.sharding import shard_range, shard_size
    n, ranks = 1500, 3
    sb, comp, _, want = pool.boundary_case(c, n=n, seed=3)
    n_shard = shard_size(n, ranks)
    with options(eng, variant, window_bits=c):
        nwin = eng.msm_window_count(n_shard)
        assert nwin == mdc.window_count(c) and eng.msm_partial_bytes(n_shard) == nwin * 160 + 8
        records = (C.c_uint64 * (20 * nwin * ranks))()
        for r in range(ranks):
            lo, hi = shard_range(n, r, ranks)
            rc, w = eng.edwards_msm_partial(sb[32 * lo:32 * hi], comp[32 * lo:32 * hi], hi - lo, n_shard)
            assert rc == 0
            C.memmove(C.addressof(records) + r * 160 * nwin, w, 160 * nwin)
        got, limbs = eng.edwards_msm_combine(records, ranks, n_shard, want_limbs=True)
    assert got == want
    assert oracle.compress(oracle.p3_from_limbs(limbs)) == want


# ---- g. widths and flat mode alternating in one context (the reduction descriptors are cached per width) ----
def test_width_switching_in_one_context(oracle, pool):
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    pre = None
    try:
        n_static = 4097
        c_flat = width_of(e, n_static)
        rnd = random.Random(20)
        sidx = [rnd.randrange(NPOOL + NTORS) for _ in range(n_static)]
        e.set_option("precomp_tables", 1)
        try:
            pre = pkg.VartimeEdwardsPrecomputation([pool.comp[j] for j in sidx], engine=e)
        finally:
            e.set_option("precomp_tables", 0)
        ss = mdc.boundary_scalars(c_flat)
        ss = ss + [rnd.getrandbits(256) for _ in range(n_static - len(ss))]
        for step, c in enumerate([20, 4, 20, "flat", 20, 4]):
            if c == "flat":
                # the static part reduces one flat window at the tables' width, the dynamic part 13 windows at c = 20
                e.set_option("window_bits", 20)
                ds =mdc.boundary_scalars(20)
                ds = ds + [rnd.getrandbits(256) for _ in range(500 - len(ds))]
                didx = [rnd.randrange(NPOOL + NTORS) for _ in range(500)]
                got = pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [b32(s) for s in ds], [pool.comp[j] for j in didx])
                assert got == pool.want(ss + ds, sidx + didx), step
            else:
                e.set_option("window_bits", c)
                sb, comp, _, want = pool.boundary_case(c, seed=step)
                rc, got, _ = e.edwards_vartime_msm(sb, comp, N_BOUNDARY)
                assert rc == 0 and got == want, step
    finally:
        if pre is not None:
            pre.close()
        e.close()


# ---- h. verification on the IMAD.WIDE field, and with the TMA gathers ----
VERIFY_VARIANTS = ["imad", "f64_tma"]


@pytest.fixture(scope="module")
def torsion_batches(oracle):
    """torsion_cases batches and the oracle's verdicts; both Ok and Verify occur"""
    out = []
    for n in (5, 100):
        for trial in range(4):
            msgs, sigs, pks = torsion_cases.make_batch(oracle, n, seed=7000 * n + trial)
            out.append((msgs, sigs, pks, oracle.verify_batch(msgs, sigs, pks)))
    assert {w for *_, w in out} == {0, 1}
    return out


@pytest.fixture(scope="module")
def validation(oracle):
    """the 914 validation vectors, flattened, with the oracle's verdicts as batches of 1 and of 32 and one by one"""
    H = bytes.fromhex
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_validation.json")) as f:
        vec = json.load(f)["vectors"]
    msgs = [v["msg"].encode() for v in vec]
    sigs = [H(v["sig"]) for v in vec]
    keys = [H(v["key"]) for v in vec]
    n = len(vec)
    batches = {bs: [oracle.verify_batch(msgs[k:k + bs], sigs[k:k + bs], keys[k:k + bs]) for k in range(0, n, bs)] for bs in (1, 32)}
    each = {strict: [oracle.verify(m, s, k, strict=strict) for m, s, k in zip(msgs, sigs, keys)] for strict in (False, True)}
    fl, offs = flat_msgs(msgs)
    return n, fl, offs, b"".join(sigs), b"".join(keys), batches, each


@pytest.mark.parametrize("variant", VERIFY_VARIANTS)
def test_verify_batch_torsion_cases(eng, torsion_batches, variant):
    with options(eng, variant):
        for k, (msgs, sigs, pks, want) in enumerate(torsion_batches):
            assert eng.verify_batch_raw(msgs, b"".join(sigs), b"".join(pks)) == want, k


@pytest.mark.parametrize("variant", VERIFY_VARIANTS)
def test_verify_batches_validation_vectors(eng, validation, variant):
    n, fl, offs, sigs, keys, batches, _ = validation
    with options(eng, variant):
        for bs, want in batches.items():
            rc, got = eng.verify_batches_flat(fl, offs, sigs, keys, n, bs)
            assert got == want, bs


@pytest.mark.parametrize("variant", VERIFY_VARIANTS)
def test_verify_each_comb_option(eng, validation, variant):
    """each_comb = 2 asks for the per-key comb tables; field_f64 = 0 falls back to the plain kernel"""
    n, fl, offs, sigs, keys, _, each = validation
    with options(eng, variant, each_comb=2):
        for strict, want in each.items():
            rc, got = eng.verify_each_flat(fl, offs, sigs, keys, n, strict=strict)
            assert got == want, strict
