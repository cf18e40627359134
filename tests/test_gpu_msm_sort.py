"""GPU tests of the two-level digit sort of the bucket MSM (k_sort_count / k_sort_bins_scan / k_sort_partition /
k_sort_fine in csrc/msm.cu) on inputs that reach its paths: coarse bins far larger than k_sort_fine holds in shared
memory, every digit of a window in one coarse bin, n around the tile sizes, flat precomputed tables, a skewed chunk
among uniform host chunks, and forced window widths.

References are exact and cheap, as in test_gpu_msm_variants.py: the points are t_j B from a pool of oracle points,
some shifted by the order-8 point T8."""
import random

import numpy as np
import pytest

import msm_digit_cases as mdc
import pyref
from test_gpu_msm_variants import NPOOL, NTORS, Pool, b32, check_msm, options, rescaled_limbs, width_of

pytestmark = pytest.mark.gpu

SORT_TILE, SORT_COUNT_TILE = 2048, 4096          # scalars per CTA of k_sort_partition and of k_sort_count


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def pool(oracle):
    return Pool(oracle)


def small_digit_scalar(rnd, c, dmax):
    """a scalar whose every signed digit at width c has magnitude <= dmax + 1: raw windows d or 2^c - d, d <= dmax,
    so a carry adds at most one to the next window"""
    s = 0
    for w in range(256 // c):
        d = rnd.randrange(1, dmax + 1)
        s |= (d if rnd.random() < 0.5 else (1 << c) - d) << (c * w)
    return s


def indices(rnd, n):
    return [NPOOL + rnd.randrange(NTORS) if i % 37 == 5 else rnd.randrange(NPOOL) for i in range(n)]


def run_host(eng, oracle, pool, scalars, idx, rnd, **opts):
    sb, comp, ext = pool.inputs(scalars, idx, rnd)
    want = pool.want(scalars, idx)
    with options(eng, **opts):
        check_msm(eng, oracle, want, sb, comp, len(scalars), point_fmt=0)
        check_msm(eng, oracle, want, sb, ext, len(scalars), point_fmt=1)


def test_all_scalars_equal(eng, oracle, pool):
    """one bucket per window: each window's coarse bin holds all 2^17 + 3 entries and takes the looped path"""
    rnd = random.Random(17)
    n = (1 << 17) + 3
    s = rnd.getrandbits(256)
    run_host(eng, oracle, pool, [s] * n, indices(rnd, n), rnd)


@pytest.mark.parametrize("n", [5000, (1 << 16) + 1])
def test_one_coarse_bin_spread_over_fine_buckets(eng, oracle, pool, n):
    """c = 16, every digit in [-65, 65]: all digits of a window fall into coarse bin 0 (at least 2^6 buckets) and
    spread over its first 65 fine buckets; 5000 entries fit in shared memory, 2^16 + 1 do not"""
    rnd = random.Random(n)
    scalars = [small_digit_scalar(rnd, 16, 64) for _ in range(n)]
    assert all(abs(d) <= 65 for s in scalars[:50] for d in mdc.signed_digits(s, 16))
    run_host(eng, oracle, pool, scalars, indices(rnd, n), rnd, window_bits=16)


@pytest.mark.parametrize("n", [1, SORT_TILE - 1, SORT_TILE, SORT_TILE + 1, SORT_COUNT_TILE - 1, SORT_COUNT_TILE,
                               SORT_COUNT_TILE + 1])
def test_sizes_around_the_tiles(eng, oracle, pool, n):
    """partial last tiles of both tiled kernels; n = 1 through the bucket pipeline (field_f64 = 0)"""
    rnd = random.Random(3 * n + 1)
    scalars = [rnd.getrandbits(256) if k % 2 else rnd.randrange(pyref.L) for k in range(n)]
    scalars[:min(n, 8)] = mdc.EDGE_SCALARS[:min(n, 8)]
    run_host(eng, oracle, pool, scalars, indices(rnd, n), rnd, variant="imad" if n < 190 else "f64")


@pytest.mark.parametrize("c", [4, 9, 16, 20])
def test_forced_widths(eng, oracle, pool, c):
    """c = 4: one bucket per coarse bin (no fine bits); c = 20: 2^12 fine buckets per coarse bin"""
    n = (1 << 16) + 1
    rnd = random.Random(c)
    scalars = mdc.boundary_scalars(c)
    scalars = scalars + [rnd.getrandbits(256) if k % 2 else rnd.randrange(pyref.L) for k in range(n - len(scalars))]
    run_host(eng, oracle, pool, scalars, indices(rnd, n), rnd, window_bits=c)


def test_flat_tables_skewed_scalars(eng, pool):
    """precomputed 2^(cw) P tables (every window counts into window 0) with a third of the scalars equal and a third
    with small digits: the coarse bins of the single bucket window are far from uniform"""
    import curve25519_dalek_b200 as pkg
    n = 4097
    c = width_of(eng, n)
    rnd = random.Random(4098)
    idx = indices(rnd, n)
    with options(eng, precomp_tables=1):
        pre = pkg.VartimeEdwardsPrecomputation([pool.comp[j] for j in idx], engine=eng)
    try:
        heavy = rnd.getrandbits(256)
        ss = [heavy if k % 3 == 0 else small_digit_scalar(rnd, c, 3) if k % 3 == 1 else rnd.getrandbits(256) for k in range(n)]
        assert pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [], []) == pool.want(ss, idx)
        ds = [heavy] * 300
        didx = indices(rnd, 300)
        got = pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [b32(s) for s in ds], [pool.comp[j] for j in didx])
        assert got == pool.want(ss + ds, idx + didx)
    finally:
        pre.close()


def test_host_chunks_one_skewed(eng, pool):
    """three host chunks: the first and last uniform, every scalar of the middle one equal"""
    n = (1 << 18) + 5
    rnd = random.Random(2185)
    scalars = [rnd.getrandbits(256) for _ in range(n)]
    heavy = rnd.getrandbits(256)
    scalars[n // 3:2 * n // 3] = [heavy] * (2 * n // 3 - n // 3)
    idx = np.array([rnd.randrange(NPOOL + NTORS) for _ in range(n)])
    sb = np.frombuffer(b"".join(b32(s) for s in scalars), dtype=np.uint8).copy()
    comp = np.frombuffer(b"".join(pool.comp), dtype=np.uint8).reshape(-1, 32)[idx].copy()
    ext = np.array([rescaled_limbs(xyzt, rnd) for xyzt in pool.xyzt], dtype=np.uint64)[idx].copy()
    want = pool.want(scalars, idx.tolist())
    with options(eng, host_chunks=3):
        for fmt, pts in ((0, comp), (1, ext)):
            rc, got, _ = eng.edwards_vartime_msm(sb, pts, n, point_fmt=fmt)
            assert rc == 0 and got == want, fmt
