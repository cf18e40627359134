"""GPU parity tests for the MSM path: the CUDA engine (through the C ABI) against the CPU oracle on
the same seeded inputs, at sizes crossing every reference threshold (SURVEY 8d config 1), plus
size-independent identities at larger n."""
import ctypes as C
import hashlib
import random

import pytest

import pyref

pytestmark = pytest.mark.gpu

SEED = 0xDA1EC00000000001


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


def gen_case(oracle, n, seed=SEED, special=True):
    """SURVEY 8(d) config 1 generators: s_i, t_i from labelled SHA-512; P_i = t_i * B."""
    B = oracle.basepoint()
    scalars, points = [], []
    for i in range(n):
        s = pyref.labelled_scalar(b"dalek-b200/scalar", seed, i)
        t = pyref.labelled_scalar(b"dalek-b200/point", seed, i)
        scalars.append(s.to_bytes(32, "little"))
        points.append(oracle.scalarmul(t.to_bytes(32, "little"), B))
    if special and n >= 8:
        # edge scalars (0, 1, l-1, 2^255-1) and edge points (identity, 8-torsion)
        scalars[0] = (0).to_bytes(32, "little")
        scalars[1] = (1).to_bytes(32, "little")
        scalars[2] = (pyref.L - 1).to_bytes(32, "little")
        scalars[3] = (2**255 - 1).to_bytes(32, "little")
        points[4] = oracle.identity()
        points[5] = oracle.decompress((0).to_bytes(32, "little"))        # order-4 point (x, 0)
        points[6] = oracle.decompress((pyref.p - 1).to_bytes(32, "little"))  # (0, -1), order 2
    return scalars, points


@pytest.mark.parametrize("n", [0, 1, 2, 3, 100, 189, 190, 250, 256, 499, 500, 799, 800, 1000])
def test_msm_parity_compressed_and_extended(eng, oracle, n):
    scalars, points = gen_case(oracle, n)
    want = oracle.compress(oracle.msm("optional", scalars, points)) if n else oracle.compress(oracle.identity())
    sb = b"".join(scalars)
    comp = b"".join(oracle.compress(p) for p in points)
    rc, got, limbs = eng.edwards_vartime_msm(sb, comp, n, point_fmt=0, want_limbs=True)
    assert rc == 0 and got == want
    # returned limbs describe the same point (projective equality, C/edwards.rs:501-512)
    assert oracle.compress(oracle.p3_from_limbs(limbs)) == want
    # extended-limb input (the reference's in-memory EdwardsPoint, Z != 1)
    ext = (C.c_uint64 * (20 * max(n, 1)))()
    for i, p in enumerate(points):
        q = oracle.add(oracle.double(p), p)            # 3p with non-trivial Z ...
        q = oracle.sub(q, oracle.double(p))            # ... back to p, Z != 1
        for k, v in enumerate(oracle.p3_limbs(q)):
            ext[20 * i + k] = v
    rc, got2, _ = eng.edwards_vartime_msm(sb, ext, n, point_fmt=1)
    assert rc == 0 and got2 == want


def test_msm_reference_kats(eng, oracle, kat):
    """multiscalar_mul_vs_ed25519py (C/edwards.rs:2428-2435) through the engine."""
    H = bytes.fromhex
    a, b = H(kat["edwards"]["A_SCALAR"]["hex"]), H(kat["edwards"]["B_SCALAR"]["hex"])
    A = H(kat["edwards"]["A_TIMES_BASEPOINT"]["hex"])
    Bc = H(kat["constants"]["ED25519_BASEPOINT_COMPRESSED"]["hex"])
    rc, got, _ = eng.edwards_vartime_msm(a + b, A + Bc, 2)
    assert rc == 0 and got == H(kat["edwards"]["DOUBLE_SCALAR_MULT_RESULT"]["hex"])
    rc, got, _ = eng.edwards_vartime_msm(a, Bc, 1)
    assert rc == 0 and got == A


def test_msm_none_on_bad_point(eng, oracle):
    scalars, points = gen_case(oracle, 20, special=False)
    comp = [oracle.compress(p) for p in points]
    comp[7] = (2).to_bytes(32, "little")              # y = 2 is not on the curve
    rc, _, _ = eng.edwards_vartime_msm(b"".join(scalars), b"".join(comp), 20)
    assert rc == 1                                     # Option::None


@pytest.mark.parametrize("bits", [4, 7, 8, 11, 13, 16])
def test_msm_every_window_width(eng, oracle, bits):
    scalars, points = gen_case(oracle, 300, seed=bits)
    want = oracle.compress(oracle.msm("optional", scalars, points))
    eng.set_option("window_bits", bits)
    try:
        rc, got, _ = eng.edwards_vartime_msm(b"".join(scalars), b"".join(oracle.compress(p) for p in points), 300)
    finally:
        eng.set_option("window_bits", 0)
    assert rc == 0 and got == want


def test_msm_skewed_buckets(eng, oracle):
    """All scalars equal: every point lands in the same bucket of each window."""
    scalars, points = gen_case(oracle, 700, special=False)
    s = scalars[0]
    want = oracle.compress(oracle.msm("optional", [s] * 700, points))
    rc, got, _ = eng.edwards_vartime_msm(s * 700, b"".join(oracle.compress(p) for p in points), 700)
    assert rc == 0 and got == want


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 17, 64, 65, 150, 189])
def test_small_msm_straus_path_and_bucket_path_agree(eng, oracle, n):
    """Below 190 points the engine follows the reference's dispatch (edwards.rs:1025-1029) to vartime Straus
    (csrc/straus_vt.cu: device non_adjacent_form(5), NafLookupTable5, straus.rs:159-200); the option `small_straus`
    switches back to the bucket pipeline.  Both must give the oracle's Straus result, for compressed and extended
    points, edge scalars, small-order points, and scalars with bit 255 set (legal at this boundary)."""
    scalars, points = gen_case(oracle, n)
    rnd = random.Random(n)
    if n >= 9:
        scalars[7] = (2**256 - 1).to_bytes(32, "little")             # beyond the reference's Scalar invariant
        scalars[8] = (2**255 + rnd.randrange(2**255)).to_bytes(32, "little")
    # oracle: the Straus algorithm itself for reference-legal scalars, exact integer arithmetic otherwise
    legal = all(int.from_bytes(x, "little") < 2**255 for x in scalars)
    if legal:
        want = oracle.compress(oracle.msm("straus_vartime", scalars, points))
        assert want == oracle.compress(oracle.msm("optional", scalars, points))
    else:
        acc = oracle.identity()
        for sc, pt in zip(scalars, points):
            v = int.from_bytes(sc, "little")
            lo = oracle.scalarmul((v % 2**252).to_bytes(32, "little"), pt)             # v = lo + 2^252 hi
            hi = oracle.mul_by_pow_2(oracle.scalarmul((v >> 252).to_bytes(32, "little"), pt), 252)
            acc = oracle.add(acc, oracle.add(lo, hi))
        want = oracle.compress(acc)
    sb = b"".join(scalars)
    comp = b"".join(oracle.compress(p) for p in points)
    ext = (C.c_uint64 * (20 * n))()
    for i, pt in enumerate(points):
        q = oracle.sub(oracle.add(oracle.double(pt), pt), oracle.double(pt))           # Z != 1
        for k, v in enumerate(oracle.p3_limbs(q)):
            ext[20 * i + k] = v
    for straus in (1, 0):
        eng.set_option("small_straus", straus)
        try:
            l0 = eng.launch_count()
            rc, got, _ = eng.edwards_vartime_msm(sb, comp, n, point_fmt=0)
            launches = eng.launch_count() - l0
            assert rc == 0 and got == want, straus
            assert (launches <= 5) == bool(straus)                   # 4 launches against ~27
            rc, got, _ = eng.edwards_vartime_msm(sb, ext, n, point_fmt=1)
            assert rc == 0 and got == want, straus
        finally:
            eng.set_option("small_straus", 1)
    # an undecodable point still gives None on the Straus path
    bad = bytearray(comp); bad[32 * (n - 1):32 * n] = (2).to_bytes(32, "little")
    rc, _, _ = eng.edwards_vartime_msm(sb, bytes(bad), n, point_fmt=0)
    assert rc == 1


def test_edwards_msm_rejects_ristretto_points(eng):
    """DALEK_POINTS_RISTRETTO (2) is a format of the Ristretto entry points only: the Edwards MSM calls reject it"""
    n = 3
    sb, pts = bytes(32 * n), bytes(32 * n)
    out = (C.c_uint8 * 32)()
    windows = (C.c_uint64 * (20 * eng.msm_window_count(n)))()
    lib, h = eng.lib, eng.h
    assert lib.dalek_b200_edwards_vartime_msm(h, sb, pts, 2, n, C.addressof(out), None) == -1
    assert lib.dalek_b200_edwards_ct_msm(h, sb, pts, 2, n, C.addressof(out), None) == -1
    assert lib.dalek_b200_edwards_msm_partial(h, sb, pts, 2, n, n, C.addressof(windows)) == -1


def test_msm_sharded_partial_combine(eng, oracle):
    """SURVEY 8(e): contiguous shards -> window accumulators -> combine == single MSM.  The window width comes from
    the SHARD size (the work one GPU does), identical on every rank."""
    from curve25519_dalek_b200.sharding import shard_range, shard_size
    n, ranks = 1203, 4
    scalars, points = gen_case(oracle, n)
    comp = [oracle.compress(p) for p in points]
    want = oracle.compress(oracle.msm("optional", scalars, points))
    n_shard = shard_size(n, ranks)
    nwin = eng.msm_window_count(n_shard)
    assert eng.msm_partial_bytes(n_shard) == nwin * 160 + 8
    allw = (C.c_uint64 * (20 * nwin * ranks))()
    for r in range(ranks):
        lo, hi = shard_range(n, r, ranks)
        rc, w = eng.edwards_msm_partial(b"".join(scalars[lo:hi]), b"".join(comp[lo:hi]), hi - lo, n_shard)
        assert rc == 0
        for k in range(20 * nwin):
            allw[r * 20 * nwin + k] = w[k]
    got, _ = eng.edwards_msm_combine(allw, ranks, n_shard)
    assert got == want


def test_msm_sharded_device_resident(eng, oracle):
    """The same exchange without leaving the device: partial_async records -> (gathered) device buffer -> combine_dev.
    Several shards are run one after another on this one GPU into slices of the gathered buffer."""
    import torch
    from curve25519_dalek_b200.sharding import shard_range, shard_size, ShardedMsm
    n, ranks = 2500, 3
    scalars, points = gen_case(oracle, n)
    comp = [oracle.compress(p) for p in points]
    want = oracle.compress(oracle.msm("optional", scalars, points))
    n_shard = shard_size(n, ranks)
    rec = eng.msm_partial_bytes(n_shard)
    dev = torch.device("cuda", 0)
    gathered = torch.zeros(ranks * rec, dtype=torch.uint8, device=dev)
    for r in range(ranks):
        lo, hi = shard_range(n, r, ranks)
        assert eng.edwards_msm_partial_async(b"".join(scalars[lo:hi]), b"".join(comp[lo:hi]), hi - lo, n_shard,
                                             gathered.data_ptr() + r * rec) == 0
    rc, got, _ = eng.edwards_msm_combine_dev(gathered.data_ptr(), ranks, n_shard)
    assert rc == 0 and got == want
    # an undecodable point in one shard marks its record: the combined result is None
    bad = list(comp); bad[n - 2] = (2).to_bytes(32, "little")         # y = 2 is not on the curve
    for r in range(ranks):
        lo, hi = shard_range(n, r, ranks)
        eng.edwards_msm_partial_async(b"".join(scalars[lo:hi]), b"".join(bad[lo:hi]), hi - lo, n_shard, gathered.data_ptr() + r * rec)
    rc, _, _ = eng.edwards_msm_combine_dev(gathered.data_ptr(), ranks, n_shard)
    assert rc == 1
    # world = 1 through the helper bench.py uses (the engine's stream as a torch ExternalStream)
    sm = ShardedMsm(eng, 1, n, dev)
    rc, got = sm.run(b"".join(scalars), b"".join(comp), n, 0, False)
    assert rc == 0 and got == want and eng.last_call_ms() > 0


def test_msm_large_algebraic_identity(eng, oracle):
    """C/edwards.rs:2281-2295 at n = 2^16: sum s_i (t_i B) == (sum s_i t_i) B, RHS by the oracle."""
    import numpy as np
    n = 1 << 16
    rnd = random.Random(1234)
    B = oracle.basepoint()
    # points: t_i * B for a small pool extended by cheap additions so the oracle cost stays low
    pool_t = [rnd.randrange(pyref.L) for _ in range(64)]
    pool_p = [oracle.compress(oracle.scalarmul(t.to_bytes(32, "little"), B)) for t in pool_t]
    idx = [rnd.randrange(64) for _ in range(n)]
    ss = [rnd.randrange(pyref.L) for _ in range(n)]
    k = sum(s * pool_t[j] for s, j in zip(ss, idx)) % pyref.L
    want = oracle.compress(oracle.scalarmul(k.to_bytes(32, "little"), B))
    sb = b"".join(s.to_bytes(32, "little") for s in ss)
    pb = b"".join(pool_p[j] for j in idx)
    rc, got, _ = eng.edwards_vartime_msm(sb, pb, n)
    assert rc == 0 and got == want


@pytest.mark.parametrize("fmt", [0, 1])
def test_msm_host_chunked_streaming(eng, oracle, fmt):
    """n = 2^18 + 5 host-buffer call: the pairs are streamed in chunks that add onto persistent bucket
    sums (copy/compute overlap); result must equal the single-shot device path and the identity
    sum s_i (t_i B) == (sum s_i t_i) B.  Skewed scalars make some buckets heavy in every chunk."""
    import numpy as np
    n = (1 << 18) + 5
    rnd = random.Random(99 + fmt)
    B = oracle.basepoint()
    pool_t = [rnd.randrange(pyref.L) for _ in range(32)]
    pool_pts = [oracle.scalarmul(t.to_bytes(32, "little"), B) for t in pool_t]
    idx = [rnd.randrange(32) for _ in range(n)]
    ss = [rnd.randrange(pyref.L) for _ in range(n)]
    for i in range(0, n, 3):
        ss[i] = ss[0]                                   # a third of the scalars are equal: heavy buckets
    k = sum(s * pool_t[j] for s, j in zip(ss, idx)) % pyref.L
    want = oracle.compress(oracle.scalarmul(k.to_bytes(32, "little"), B))
    sb = np.frombuffer(b"".join(s.to_bytes(32, "little") for s in ss), dtype=np.uint8).copy()
    if fmt == 0:
        enc = [oracle.compress(p) for p in pool_pts]
        pb = np.frombuffer(b"".join(enc[j] for j in idx), dtype=np.uint8).copy()
    else:
        lim = [np.array(oracle.p3_limbs(oracle.add(oracle.double(p), p)), dtype=np.uint64) for p in pool_pts]   # 3P, Z != 1
        pb = np.stack([lim[j] for j in idx]).copy()
        k = 3 * k % pyref.L
        want = oracle.compress(oracle.scalarmul(k.to_bytes(32, "little"), B))
    for chunks in (4, 1, 3):
        eng.set_option("host_chunks", chunks)
        try:
            rc, got, _ = eng.edwards_vartime_msm(sb, pb, n, point_fmt=fmt)
        finally:
            eng.set_option("host_chunks", 8)                # the engine's default
        assert rc == 0 and got == want, chunks


@pytest.mark.parametrize("f64", [1, 0])
def test_decompress_edge_encodings(eng, oracle, kat, f64):
    """CompressedEdwardsY::decompress (C/edwards.rs:211-257) inside the engine, with the square-root exponentiation
    on either field: 1*P for edge encodings (non-canonical y, sign bit on x = 0, small order, non-squares) must
    give the oracle's Option -- None, or the canonical re-encoding of the same point."""
    p = pyref.p
    rnd = random.Random(99)
    encs = [y.to_bytes(32, "little") for y in (0, 1, 2, 3, 4, 5, p - 1, p, p + 1, p + 2, 2**255 - 1, 2**255 - 20, 2**254, 19)]
    encs += [(y | (1 << 255)).to_bytes(32, "little") for y in (0, 1, p - 1, p, p + 1, 2**255 - 1, 4)]
    encs += [bytes.fromhex(h) for h in (                      # order-8 points and their negatives
        "26e8958fc2b227b045c3f489f2ef98f0d5dfac05d3c63339b13802886d53fc05", "26e8958fc2b227b045c3f489f2ef98f0d5dfac05d3c63339b13802886d53fc85",
        "c7176a703d4dd84fba3c0b760d10670f2a2053fa2c39ccc64ec7fd7792ac037a", "c7176a703d4dd84fba3c0b760d10670f2a2053fa2c39ccc64ec7fd7792ac03fa")]
    encs += [rnd.randbytes(32) for _ in range(60)]
    one = (1).to_bytes(32, "little")
    eng.set_option("decompress_f64", f64)
    try:
        n_none = 0
        for e in encs:
            q = oracle.decompress(e)
            rc, got, _ = eng.edwards_vartime_msm(one, e, 1)
            if q is None:
                assert rc == 1, e.hex()
                n_none += 1
            else:
                assert rc == 0 and got == oracle.compress(q), e.hex()
        assert 10 < n_none < len(encs) - 10
        # and all of the decodable ones in one call: sum_i (i+1) * P_i
        good = [e for e in encs if oracle.decompress(e) is not None]
        sc = [(i + 1).to_bytes(32, "little") for i in range(len(good))]
        want = oracle.compress(oracle.msm("optional", sc, [oracle.decompress(e) for e in good]))
        rc, got, _ = eng.edwards_vartime_msm(b"".join(sc), b"".join(good), len(good))
        assert rc == 0 and got == want
    finally:
        eng.set_option("decompress_f64", 1)
