"""GPU parity tests for the three passes that normalise extended input points to Z = 1 (csrc/msm.cu): k_prep_zprod
multiplies the Z of each group of GROUP points, k_prep_invert inverts all the group products in one CTA of THREADS
threads with one field inversion (each thread takes a run of products when there are more groups than threads), and
k_prep_finish recovers every 1/Z from its group's inverse.  The sizes straddle the warp, the group and the width of
k_prep_invert's CTA; points with Z = 0 (mod p) sit at the first and last point of a thread, a warp, a group and the
input, and must become the identity without disturbing the rest of their group.  Every point carries its own
projective scale lambda; results are checked against the C oracle."""
import random
from contextlib import contextmanager

import numpy as np
import pytest

import pyref

pytestmark = pytest.mark.gpu

GROUP = 1024                                  # PREP_GROUP: points per group product
THREADS = 256                                 # PREP_THREADS: threads per CTA of the three passes
PER_THREAD = GROUP // THREADS                 # point k of thread t in a group: k * THREADS + t
MASK51 = (1 << 51) - 1
P_LIMBS = [MASK51 - 18, MASK51, MASK51, MASK51, MASK51]   # p itself: Z = 0 mod p with non-zero limbs


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@contextmanager
def options(eng, **kv):
    try:
        for k, v in kv.items():
            eng.set_option(k, v)
        yield
    finally:
        eng.set_option("small_straus", 1)      # the engine's defaults
        eng.set_option("host_chunks", 8)


def b32(x):
    return x.to_bytes(32, "little")


def limbs_of(vals):
    return [(v >> (51 * k)) & MASK51 for v in vals for k in range(5)]


def rescaled(oracle, p, lam):
    """(lambda X : lambda Y : lambda Z : lambda T) of p as 20 radix-2^51 limbs"""
    lim = oracle.p3_limbs(p)
    xyzt = [sum(lim[5 * c + k] << (51 * k) for k in range(5)) % pyref.p for c in range(4)]
    return limbs_of([v * lam % pyref.p for v in xyzt])


@pytest.fixture(scope="module")
def pool(oracle):
    """64 multiples t B, each under four scales; the specials (identity and two torsion points) under two each"""
    rnd = random.Random(0x9E3)
    B = oracle.basepoint()
    rows, logs = [], []
    for _ in range(64):
        t = rnd.randrange(1, pyref.L)
        p = oracle.scalarmul(b32(t), B)
        for _ in range(4):
            rows.append(rescaled(oracle, p, rnd.randrange(2, pyref.p))); logs.append(t)
    specials = [oracle.identity(), oracle.decompress(b32(0)), oracle.decompress(b32(pyref.p - 1))]
    sp_rows = [rescaled(oracle, s, lam) for s in specials for lam in (pyref.p - 1, rnd.randrange(2, pyref.p))]
    sp_pts = [s for s in specials for _ in range(2)]
    return np.array(rows, dtype=np.uint64), logs, np.array(sp_rows, dtype=np.uint64), sp_pts


def make_case(oracle, pool, n, seed, zeros=(), specials=()):
    """n pairs: scalars below 2^252, pool points; Z = 0 at `zeros` (alternately all-zero limbs and the limbs of p),
    pool specials at `specials`.  Returns (scalars n x 32 u8, points n x 20 u64, the expected compressed result)."""
    rows, logs, sp_rows, sp_pts = pool
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(logs), n)
    ext = rows[idx].copy()
    sc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sc[:, 31] &= 0x0F
    zeros, specials = sorted(set(zeros)), sorted(set(specials) - set(zeros))
    skip = set(zeros) | set(specials)
    k = 0
    for i in range(n):
        if i not in skip:
            k += int.from_bytes(sc[i].tobytes(), "little") * logs[idx[i]]
    want = oracle.scalarmul(b32(k % pyref.L), oracle.basepoint())
    for j, i in enumerate(specials):
        ext[i] = sp_rows[j % len(sp_rows)]
        want = oracle.add(want, oracle.scalarmul(sc[i].tobytes(), sp_pts[j % len(sp_pts)]))
    for j, i in enumerate(zeros):                  # not a point: it must count as the identity, whatever its scalar
        ext[i, 10:15] = P_LIMBS if j & 1 else 0
    return sc, ext, oracle.compress(want)


def msm_all_paths(eng, sc, ext, n, want, host_chunks=(8,)):
    """The bucket pipeline (vartime Straus off, so that small n take the three passes too) from device-resident inputs
    and from host buffers"""
    import torch
    dev = torch.device("cuda", 0)
    d_s = torch.from_numpy(sc.reshape(-1)).to(dev)
    d_p = torch.from_numpy(ext.reshape(-1).view(np.uint8)).to(dev)
    torch.cuda.synchronize()
    with options(eng, small_straus=0):
        rc, got, _ = eng.edwards_vartime_msm(d_s.data_ptr(), d_p.data_ptr(), n, point_fmt=1, device_ptrs=True)
        assert (rc, got) == (0, want), "device-resident"
        for chunks in host_chunks:
            eng.set_option("host_chunks", chunks)
            rc, got, _ = eng.edwards_vartime_msm(sc, ext, n, point_fmt=1)
            assert (rc, got) == (0, want), "host buffers, %d chunks" % chunks


def groups(n):
    return (n + GROUP - 1) // GROUP


SIZES = [1, 2, 31, 32, 33, GROUP - 1, GROUP, GROUP + 1,
         2 * GROUP,                           # two groups
         3 * GROUP - 5,                       # three, the last one short
         (THREADS - 1) * GROUP,               # k_prep_invert: one group per thread but the last
         THREADS * GROUP,                     # one group per thread
         THREADS * GROUP + 1,                 # THREADS + 1 groups: thread 0 of k_prep_invert takes two
         (2 * THREADS + 1) * GROUP - 300]     # 2 THREADS + 1 groups: runs of three products, the last ones short


@pytest.mark.parametrize("n", SIZES)
def test_sizes(eng, oracle, pool, n):
    specials = [i for g in range(0, n + 1, GROUP) for i in (g - 1, g, g + 1) if 0 <= i < n] if n > 32 else []
    sc, ext, want = make_case(oracle, pool, n, seed=n, specials=specials)
    msm_all_paths(eng, sc, ext, n, want)


def test_group_counts():
    """SIZES reach the group counts the passes branch on"""
    g = {groups(n) for n in SIZES}
    assert {1, 2, 3, THREADS - 1, THREADS, THREADS + 1, 2 * THREADS + 1} <= g


def zero_positions(n_groups):
    """Z = 0 at the first and last point of a thread, of a warp, of a group, and all of group 3"""
    thread = [GROUP + 5, GROUP + (PER_THREAD - 1) * THREADS + 5]                # thread 5 of group 1
    warp = [64, (PER_THREAD - 1) * THREADS + 95]                                 # warp 2 of group 0
    lanes = [2 * GROUP + 32 * w + l for w in range(THREADS // 32) for l in (0, 31)]   # each warp's lanes 0, 31 (k = 0)
    group = [2 * GROUP, 3 * GROUP - 1]
    whole = list(range(3 * GROUP, 4 * GROUP))
    assert n_groups > 4
    return thread + warp + lanes + group + whole


@pytest.mark.parametrize("n", [5 * GROUP, 5 * GROUP + 77])
def test_zero_z(eng, oracle, pool, n):
    zeros = zero_positions(groups(n)) + [0, n - 1]
    sc, ext, want = make_case(oracle, pool, n, seed=3 * n, zeros=zeros, specials=[1, GROUP, n - 2])
    msm_all_paths(eng, sc, ext, n, want)


@pytest.mark.parametrize("n", [1, 33, GROUP + 1])
def test_all_z_zero(eng, oracle, pool, n):
    sc, ext, want = make_case(oracle, pool, n, seed=5 * n, zeros=range(n))
    assert want == oracle.compress(oracle.identity())
    msm_all_paths(eng, sc, ext, n, want)


def test_host_chunks_split_groups(eng, oracle, pool):
    """Host buffers of 2^18 + 333 pairs in 3, 5 and 8 chunks: no chunk boundary falls on a group boundary, and Z = 0
    sits on both sides of each"""
    n = (1 << 18) + 333
    cuts = [n * k // K for K in (3, 5, 8) for k in range(1, K)]
    assert all(c % GROUP for c in cuts)
    zeros = [c + d for c in cuts for d in (-1, 0)]
    sc, ext, want = make_case(oracle, pool, n, seed=11, zeros=zeros, specials=[c + 1 for c in cuts])
    msm_all_paths(eng, sc, ext, n, want, host_chunks=(3, 5, 8))


def test_precomputation_from_extended_points(eng, oracle, pool):
    """dalek_b200_precomp_new over extended points prepares them with the same passes: its MSM equals the plain one"""
    import curve25519_dalek_b200 as pkg
    n = 5 * GROUP + 3
    sc, ext, want = make_case(oracle, pool, n, seed=13, specials=[0, GROUP - 1, GROUP, n - 1])
    scalars = [sc[i].tobytes() for i in range(n)]
    pre = pkg.VartimeEdwardsPrecomputation((ext, n), engine=eng, fmt=pkg.POINTS_EXTENDED)
    try:
        got_pre = pre.vartime_multiscalar_mul(scalars)
    finally:
        pre.close()
    rc, got, _ = eng.edwards_vartime_msm(sc, ext, n, point_fmt=1)
    assert rc == 0 and got_pre == got == want
