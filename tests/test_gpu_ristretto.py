"""GPU tests of the Ristretto entry points: every rejection term at every decode site, coset invariance of the
encoder, and the vartime MSM at every size class and bucket-kernel form.

The engine decodes CompressedRistretto (ristretto.rs:266-345) in four places: ristretto_decompress_batch
(k_ristretto_decompress_batch), the vartime MSM and the precomputation's static and dynamic points (k_prep_ristretto),
and G / H of the double-base batch.  Both kernels compile the square root for both fields (option decompress_f64);
the double-base decode always runs on the integer field.
tests/golden/ristretto.json holds vectors that fire each of the five rejection terms alone; each one is placed at the
first, the middle and the last slot of an otherwise valid input.

The encoder (ristretto.rs:500-533) picks rotate and the signs from the representative it is given, so the same
Ristretto point is fed as P + T for every T of the 4-torsion, with Z != 1.  Like the Edwards MSM, the Ristretto MSM
runs vartime Straus below 190 pairs when small_straus = 1 and field_f64 = 1; the size test also runs with
small_straus = 0, so that the bucket pipeline still runs on nearly empty windows.  The MSM points are t_j B, and the group has prime order l, so the expected result of sum s_i P_i is encode(((sum s_i t_i) mod l) B)
for any 256-bit scalars."""
import contextlib
import json
import os
import random

import numpy as np
import pytest

import msm_digit_cases as mdc
import pyref
from test_gpu_msm_affine_prep import coords, limbs_of
from test_gpu_msm_variants import VARIANTS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L
DEFAULTS = dict(field_f64=1, acc_tma=0, window_bits=0, decompress_f64=1, double_base_comb=1, small_straus=1)
NPOOL = 64
EDGES = [2**256 - 1, L + 1, 1, L - 1, 2**255 - 1, 2**252, L, 0]      # nonzero first, so that n = 1 .. 3 are not trivial
E4 = (0, 2, 4, 6)                 # EIGHT_TORSION[2k] (u64/constants.rs): the identity and the points of E[4]


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@contextlib.contextmanager
def options(eng, **opts):
    """the options for the body of the block; all of them are reset to the engine's defaults afterwards"""
    try:
        for k, v in opts.items():
            eng.set_option(k, v)
        yield
    finally:
        for k in opts:
            eng.set_option(k, DEFAULTS[k])


def form(variant):
    field_f64, acc_tma = VARIANTS[variant]
    return dict(field_f64=field_f64, acc_tma=acc_tma)


def b32(x):
    return x.to_bytes(32, "little")


@pytest.fixture(scope="module")
def golden():
    """(bad, valid): bad = [(label, encoding)] with every vector of the fixture that has a rejection term"""
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        doc = json.load(f)
    bad, valid = [], []
    for name, vs in doc["classes"].items():
        for v in vs:
            enc = bytes.fromhex(v["s"])
            if v["terms"]:
                bad.append(("%s %s %s" % (name, "+".join(v["terms"]), v["s"]), enc))
            else:
                valid.append(enc)
    assert len(bad) > 80 and len(valid) == 32
    return bad, valid


class Pool:
    """NPOOL points t_j B as Ristretto encodings, and MSM cases over them"""

    def __init__(self, oracle):
        self.oracle = oracle
        rnd = random.Random(0x8E57)
        self.B = oracle.basepoint()
        self.t = [rnd.randrange(1, L) for _ in range(NPOOL)]
        self.enc = [oracle.ristretto_compress(oracle.scalarmul(b32(t), self.B)) for t in self.t]
        self.enc_np = np.frombuffer(b"".join(self.enc), dtype=np.uint8).reshape(NPOOL, 32)
        self.cases = {}

    def encode(self, k):
        """the Ristretto encoding of (k mod l) B"""
        return self.oracle.ristretto_compress(self.oracle.scalarmul(b32(k % L), self.B))

    def want(self, scalars, idx):
        return self.encode(sum(s * self.t[j] for s, j in zip(scalars, idx)))

    def case(self, n, seed=0):
        """(scalar bytes, point bytes, scalars, idx, want): the edge scalars first, then random scalars below l and
        up to 2^256 - 1; every fifth point repeats its predecessor"""
        key = (n, seed)
        if key not in self.cases:
            rnd = random.Random(1000 * n + seed)
            scalars = EDGES[:n] + [rnd.getrandbits(256) if k % 2 else rnd.randrange(L) for k in range(n - len(EDGES))]
            idx = [rnd.randrange(NPOOL) for _ in range(n)]
            for i in range(5, n, 5):
                idx[i] = idx[i - 1]
            sb = np.frombuffer(b"".join(b32(s) for s in scalars), dtype=np.uint8).copy()
            pts = self.enc_np[np.array(idx, dtype=np.int64)].copy() if n else np.zeros(32, dtype=np.uint8)
            self.cases[key] = (sb, pts, scalars, idx, self.want(scalars, idx))
        return self.cases[key]


@pytest.fixture(scope="module")
def pool(oracle):
    return Pool(oracle)


def with_bad(valid, n, pos, bad):
    encs = [valid[k % len(valid)] for k in range(n)]
    encs[pos] = bad
    return encs


# ---- 1. every rejection term at every decode site ----
N_SITE = 9
POSITIONS = (0, N_SITE // 2, N_SITE - 1)


@pytest.mark.parametrize("f64", [1, 0])
def test_decompress_batch_rejections(eng, oracle, golden, f64):
    bad, valid = golden
    n = N_SITE
    with options(eng, decompress_f64=f64):
        for label, enc in bad:
            for pos in POSITIONS:
                encs = with_bad(valid, n, pos, enc)
                rc, limbs, ok = eng.decompress_batch(b"".join(encs), n, ristretto=True)
                assert rc == 1 and ok == bytes(int(i != pos) for i in range(n)), (label, pos)
                for i in range(n):
                    if i != pos:
                        assert oracle.ristretto_compress(oracle.p3_from_limbs(list(limbs[20 * i:20 * i + 20]))) == encs[i]
        # every vector of the fixture in one call: the exact ok flags
        encs = [e for _, e in bad] + valid
        rc, limbs, ok = eng.decompress_batch(b"".join(encs), len(encs), ristretto=True)
        assert rc == 1 and ok == bytes([0] * len(bad) + [1] * len(valid))


@pytest.mark.parametrize("f64", [1, 0])
def test_vartime_msm_rejections(eng, oracle, golden, f64):
    bad, valid = golden
    n = N_SITE
    rnd = random.Random(f64)
    sb = b"".join(b32(rnd.randrange(L)) for _ in range(n))
    with options(eng, decompress_f64=f64):
        encs = [valid[k % len(valid)] for k in range(n)]
        rc, got = eng.ristretto_vartime_msm(sb, b"".join(encs), n)
        P = [oracle.ristretto_decompress(e) for e in encs]
        want = oracle.ristretto_compress(oracle.msm("optional", [sb[32 * i:32 * i + 32] for i in range(n)], P))
        assert rc == 0 and got == want
        for label, enc in bad:
            for pos in POSITIONS:
                rc, _ = eng.ristretto_vartime_msm(sb, b"".join(with_bad(valid, n, pos, enc)), n)
                assert rc == 1, (label, pos)


@pytest.mark.parametrize("f64", [1, 0])
def test_precomputation_rejections(eng, pool, golden, f64):
    """a bad static point makes the constructor raise; a bad dynamic point makes the result None"""
    import curve25519_dalek_b200 as pkg
    bad, _ = golden
    n = N_SITE
    rnd = random.Random(10 + f64)
    sidx = [rnd.randrange(NPOOL) for _ in range(n)]
    didx = [rnd.randrange(NPOOL) for _ in range(n)]
    ss = [rnd.randrange(L) for _ in range(n)]
    ds = [rnd.randrange(L) for _ in range(n)]
    static = [pool.enc[j] for j in sidx]
    dynamic = [pool.enc[j] for j in didx]
    with options(eng, decompress_f64=f64):
        pre = pkg.VartimeRistrettoPrecomputation(static, engine=eng)
        try:
            got = pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [b32(s) for s in ds], dynamic)
            assert got == pool.want(ss + ds, sidx + didx)
            for label, enc in bad:
                for pos in POSITIONS:
                    with pytest.raises(ValueError):
                        pkg.VartimeRistrettoPrecomputation(with_bad(static, n, pos, enc), engine=eng)
                    got = pre.optional_mixed_multiscalar_mul([b32(s) for s in ss], [b32(s) for s in ds],
                                                             with_bad(dynamic, n, pos, enc))
                    assert got is None, (label, pos)
        finally:
            pre.close()


@pytest.mark.parametrize("comb", [0, 1])
@pytest.mark.parametrize("n", [4095, 4096])
def test_double_base_rejections(eng, oracle, pool, golden, n, comb):
    """G and H are decoded once per call on the integer field, by k_double_base_tables or, with double_base_comb = 1
    and n >= 4096, by every thread of k_comb_tables"""
    bad, _ = golden
    rnd = random.Random(n + comb)
    a = b"".join(b32(rnd.randrange(L)) for _ in range(n))
    b = b"".join(b32(rnd.randrange(L)) for _ in range(n))
    G, H = pool.enc[0], pool.enc[1]
    with options(eng, double_base_comb=comb):
        rc, out = eng.ristretto_double_base_batch(a, b, G, H, n)
        k = 8
        assert rc == 0 and out[-32 * k:] == oracle.ristretto_double_base_batch(a[-32 * k:], b[-32 * k:], G, H)[1]
        for label, enc in bad:
            assert eng.ristretto_double_base_batch(a, b, enc, H, n)[0] == 1, ("G", label)
            assert eng.ristretto_double_base_batch(a, b, G, enc, n)[0] == 1, ("H", label)


# ---- 2. one encoding per coset P + E[4], from representatives with Z != 1 ----
@pytest.fixture(scope="module")
def cosets(oracle, kat):
    """[(P, t, [limbs of lambda (P + T) for T in E[4]])] for the identity and 64 random P = t B"""
    tl = kat["u64_constants"]["EIGHT_TORSION_XYZT"]["limbs"]
    tors = [oracle.p3_from_limbs(tl[20 * i:20 * i + 20]) for i in E4]
    assert oracle.is_identity(tors[0]) and all(oracle.is_identity(oracle.mul_by_pow_2(T, 2)) for T in tors)
    rnd = random.Random(0xC05E7)
    B = oracle.basepoint()
    out = []
    for t in [0] + [rnd.randrange(1, L) for _ in range(64)]:
        P = oracle.scalarmul(b32(t), B)
        members = []
        for T in tors:
            lam = rnd.randrange(2, pyref.p)
            members.append(limbs_of([v * lam % pyref.p for v in coords(oracle.p3_limbs(oracle.add(P, T)))]))
        out.append((P, t, members))
    return out


def test_double_and_compress_coset_invariance(eng, oracle, cosets):
    limbs = np.array([m for _, _, ms in cosets for m in ms], dtype=np.uint64)
    got = eng.ristretto_double_and_compress_batch(limbs, len(limbs))
    for j, (P, t, _) in enumerate(cosets):
        want = oracle.ristretto_compress(oracle.double(P))
        for k in range(len(E4)):
            assert got[32 * (4 * j + k):32 * (4 * j + k + 1)] == want, (t, k)


@pytest.mark.parametrize("n_static", [0, 3])
def test_precomputation_extended_dynamic_coset_invariance(eng, oracle, pool, cosets, n_static):
    """one dynamic point with an odd scalar, so that s (P + T) runs through the whole coset of s P"""
    import curve25519_dalek_b200 as pkg
    pre = pkg.VartimeRistrettoPrecomputation(pool.enc[:3], engine=eng)
    rnd = random.Random(n_static)
    try:
        for P, t, members in cosets:
            ss = [rnd.randrange(L) for _ in range(n_static)]
            s = rnd.randrange(L) | 1
            want = pool.encode(sum(a * u for a, u in zip(ss, pool.t)) + s * t)
            sb = [b32(a) for a in ss]
            assert pre.optional_mixed_multiscalar_mul(sb, [b32(s)], [oracle.ristretto_compress(P)]) == want, t
            for k, m in enumerate(members):
                got = pre.optional_mixed_multiscalar_mul(sb, [b32(s)], [np.array(m, dtype=np.uint64).tobytes()],
                                                         dynamic_fmt=pkg.POINTS_EXTENDED)
                assert got == want, (t, k)
    finally:
        pre.close()


# ---- 3. the vartime MSM by size, bucket-kernel form, decode field and small-input path ----
SIZES = [0, 1, 2, 3, 17, 189, 190, 191, 1000]


@pytest.mark.parametrize("small_straus", [1, 0])
@pytest.mark.parametrize("f64", [1, 0])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("n", SIZES)
def test_vartime_msm_sizes_and_forms(eng, oracle, pool, n, variant, f64, small_straus):
    sb, pts, scalars, idx, want = pool.case(n)
    if n <= 191 and (variant, f64, small_straus) == ("f64", 1, 1):
        # the oracle's own MSM on the decoded points agrees (scalars reduced: the group has order l)
        P = [oracle.ristretto_decompress(pool.enc[j]) for j in idx]
        got = oracle.msm("optional", [b32(s % L) for s in scalars], P)
        assert oracle.ristretto_compress(got) == want
    with options(eng, decompress_f64=f64, small_straus=small_straus, **form(variant)):
        rc, got = eng.ristretto_vartime_msm(sb, pts, n)
    assert rc == 0 and got == want


@pytest.mark.parametrize("c", range(4, 21))
def test_vartime_msm_every_window_width(eng, pool, c):
    n = 3001
    sb, pts, _, _, want = pool.case(n)
    with options(eng, window_bits=c):
        assert eng.msm_window_count(n) == mdc.window_count(c)
        rc, got = eng.ristretto_vartime_msm(sb, pts, n)
    assert rc == 0 and got == want


def test_vartime_msm_large(eng, pool):
    """2^18 + 3 pairs: the host inputs are streamed in chunks"""
    for n in ((1 << 16) + 3, (1 << 18) + 3):
        sb, pts, _, _, want = pool.case(n)
        rc, got = eng.ristretto_vartime_msm(sb, pts, n)
        assert rc == 0 and got == want, n


# ---- 4. results equal to the identity encode as 32 zero bytes ----
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_identity_results_encode_as_zero(eng, pool, variant):
    rnd = random.Random(len(variant))
    zero = bytes(32)
    cases = [("empty", b"", b"", 0)]
    idx = [rnd.randrange(NPOOL) for _ in range(300)]
    for n in (5, 300):
        cases.append(("zero scalars", bytes(32 * n), b"".join(pool.enc[j] for j in idx[:n]), n))
    for n in (1, 150):                                      # n pairs: 2, 300 points
        ss, pts = [], []
        for j in idx[:n]:
            a = rnd.randrange(1, L)
            ss += [a, a]
            pts += [pool.enc[j], pool.encode(-pool.t[j])]    # P and -P, equal scalars
        cases.append(("P, -P", b"".join(b32(s) for s in ss), b"".join(pts), 2 * n))
        ss, pts = [], []
        for j in idx[:n]:
            a = rnd.randrange(1, L)
            ss += [a, L - a]
            pts += [pool.enc[j], pool.enc[j]]                # P and P, scalars a and l - a
        cases.append(("P, P", b"".join(b32(s) for s in ss), b"".join(pts), 2 * n))
    for f64 in (1, 0):
        with options(eng, decompress_f64=f64, **form(variant)):
            for name, sb, pb, n in cases:
                rc, got = eng.ristretto_vartime_msm(sb, pb, n)
                assert rc == 0 and got == zero, (name, n, f64)
