"""GPU parity tests for the preparation of extended input points: every point is normalised to Z = 1 (affine Niels)
with one batched inversion per group of 1024 points (PREP_GROUP in csrc/msm.cu) before the bucket kernel.  The
inputs here carry an arbitrary projective scale (lambda X : lambda Y : lambda Z : lambda T), the sizes straddle the
group size, and special points sit at the group boundaries."""
import ctypes as C
import random

import pytest

import pyref

pytestmark = pytest.mark.gpu

GROUP = 1024                                  # points sharing one inversion in the extended-point preparation
MASK51 = (1 << 51) - 1


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


def b32(x):
    return x.to_bytes(32, "little")


def coords(limbs):
    """20 radix-2^51 limbs -> (X, Y, Z, T) as integers mod p"""
    return [sum(limbs[5 * c + k] << (51 * k) for k in range(5)) % pyref.p for c in range(4)]


def limbs_of(xyzt):
    return [(v >> (51 * k)) & MASK51 for v in xyzt for k in range(5)]


def case(oracle, n, seed):
    """n terms; identity and torsion points at the group boundaries, every point rescaled by its own lambda != 0"""
    rnd = random.Random(seed)
    B = oracle.basepoint()
    points = [oracle.scalarmul(b32(rnd.randrange(1, pyref.L)), B) for _ in range(n)]
    scalars = [b32(rnd.randrange(pyref.L)) for _ in range(n)]
    specials = [oracle.identity(), oracle.decompress(b32(0)), oracle.decompress(b32(pyref.p - 1))]
    for j, g in enumerate(range(0, n + 1, GROUP)):
        for i, p in zip((g - 1, g, g + 1), specials[j % 3:] + specials[:j % 3]):
            if 0 <= i < n:
                points[i] = p
    if n:
        points[n - 1] = specials[1]
    ext = (C.c_uint64 * (20 * max(n, 1)))()
    for i, p in enumerate(points):
        lam = (1, pyref.p - 1)[i] if i < 2 else rnd.randrange(2, pyref.p)
        xyzt = [v * lam % pyref.p for v in coords(oracle.p3_limbs(p))]
        for k, v in enumerate(limbs_of(xyzt)):
            ext[20 * i + k] = v
    return scalars, points, ext


@pytest.mark.parametrize("n", [GROUP - 1, GROUP, GROUP + 1, 3 * GROUP + 77])
def test_msm_rescaled_extended_points(eng, oracle, n):
    scalars, points, ext = case(oracle, n, seed=n)
    want = oracle.compress(oracle.msm("optional", scalars, points))
    sb = b"".join(scalars)
    rc, got, _ = eng.edwards_vartime_msm(sb, ext, n, point_fmt=1)
    assert rc == 0 and got == want
    # compressed input of the same points gives the same encoding
    rc, got_c, _ = eng.edwards_vartime_msm(sb, b"".join(oracle.compress(p) for p in points), n, point_fmt=0)
    assert rc == 0 and got_c == want
    # device-resident inputs: the preparation runs on the second stream under the digit sort
    import torch
    dev = torch.device("cuda", 0)
    d_s = torch.frombuffer(bytearray(sb), dtype=torch.uint8).to(dev)
    d_p = torch.frombuffer(bytearray(bytes(ext)), dtype=torch.uint8).to(dev)
    torch.cuda.synchronize()
    rc, got_d, _ = eng.edwards_vartime_msm(d_s.data_ptr(), d_p.data_ptr(), n, point_fmt=1, device_ptrs=True)
    assert rc == 0 and got_d == want


def test_precomputed_rescaled_extended_points(eng, oracle):
    import curve25519_dalek_b200 as pkg
    n_s, n_d = GROUP + 1, GROUP - 1
    ss, sp, sext = case(oracle, n_s, seed=7)
    ds, dp, dext = case(oracle, n_d, seed=8)
    want = oracle.compress(oracle.msm("optional", ss + ds, sp + dp))
    pre = pkg.VartimeEdwardsPrecomputation((sext, n_s), engine=eng, fmt=pkg.POINTS_EXTENDED)
    assert pre.optional_mixed_multiscalar_mul(ss, ds, [bytes(dext)[160 * i:160 * (i + 1)] for i in range(n_d)],
                                              dynamic_fmt=pkg.POINTS_EXTENDED) == want
    pre.close()


def test_zero_z_does_not_disturb_its_group(eng, oracle):
    """Z = 0 is not a point (a caller's bad limbs).  Its own contribution is unspecified; the other points of its
    inversion group must still count exactly, and the call must not fail."""
    n = GROUP + 3
    scalars, points, ext = case(oracle, n, seed=99)
    for i in (5, GROUP - 1):                         # one inside the first group, one at its last position
        for k in range(20):
            ext[20 * i + k] = 1 if k == 5 else 0      # (0 : 1 : 0 : 0)
        scalars[i] = b32(0)
    want = oracle.compress(oracle.msm("optional", [s for i, s in enumerate(scalars) if i not in (5, GROUP - 1)],
                                      [p for i, p in enumerate(points) if i not in (5, GROUP - 1)]))
    rc, got, _ = eng.edwards_vartime_msm(b"".join(scalars), ext, n, point_fmt=1)
    assert rc == 0 and got == want
