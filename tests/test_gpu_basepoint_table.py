"""GPU resident basepoint tables: dalek_b200_basepoint_tables_new / _basepoints / _mul / _mul_dev and the Python
EdwardsBasepointTable / RistrettoBasepointTable (BasepointTable, C/traits.rs:50-74), against the C oracle and against
dalek_b200_mul_batch on the same inputs."""
import array
import ctypes as C
import random
import threading

import pytest

import oracle_lib
import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

L = pyref.L
P25519 = 2**255 - 19
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
DALEK_NONE, INVALID = 1, -1
PIECE = 1 << 16


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng2():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


def b32(x):
    return x.to_bytes(32, "little")


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()


def clamp(b):
    b = bytearray(b)
    b[0] &= 248
    b[31] &= 127
    b[31] |= 64
    return bytes(b)


def encode(orc, P, fmt):
    return orc.ristretto_compress(P) if fmt == RISTRETTO else orc.compress(P)


def point_input(orc, P, fmt):
    if fmt == EXTENDED:
        return b"".join(int(v).to_bytes(8, "little") for v in orc.p3_limbs(P))
    return encode(orc, P, fmt)


def want(orc, s, P, fmt, clamped=False):
    return encode(orc, orc.scalarmul(clamp(s) if clamped else s, P), fmt)


def random_points(orc, rnd, k):
    B = orc.basepoint()
    return [orc.scalarmul(b32(rnd.randrange(1, L)), B) for _ in range(k)]


def edge_scalars(rnd):
    return [0, 1, L - 1, L, L + 1, 2**255 - 1, 2**253 + 7, rnd.randrange(L, 2**255), rnd.randrange(L, 2**255),
            rnd.randrange(L), rnd.randrange(L), rnd.randrange(2**255)]


class Tables:
    """A handle of the C ABI, destroyed on exit."""

    def __init__(self, eng, inputs, fmt):
        self.eng = eng
        rc, self.h, self.ok = eng.basepoint_tables_new(b"".join(inputs), len(inputs), fmt)
        assert rc == 0 and self.ok == b"\x01" * len(inputs)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.eng.basepoint_tables_destroy(self.h)

    def mul(self, ss, idx=None, device=False, clamped=False):
        n = len(ss)
        ib = array.array("I", idx).tobytes() if idx is not None else None
        if device:
            out = self.eng.basepoint_tables_mul(self.h, dev(b"".join(ss)), dev(ib) if ib is not None else None, n,
                                                clamped=clamped, device_ptrs=True)
            return split(bytes(out.cpu().numpy())[:32 * n])
        return split(self.eng.basepoint_tables_mul(self.h, b"".join(ss), ib, n, clamped=clamped))


def mul_batch_each(eng, ss, inputs, fmt, clamped=False):
    """mul_batch with one point per item: what the tables must reproduce byte for byte"""
    n = len(ss)
    rc, out, _ = eng.mul_batch(b"".join(ss), n, b"".join(inputs), n, n, fmt, clamped=clamped)
    assert rc == 0
    return split(out)


@pytest.mark.parametrize("fmt", [COMPRESSED, EXTENDED, RISTRETTO])
@pytest.mark.parametrize("n", [1, 7, 1000])
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_formats_one_table_and_indices(eng, orc, fmt, n, device, indexed):
    rnd = random.Random(1000 * fmt + 10 * n + 2 * device + indexed)
    k = 3 if indexed else 1
    pts = random_points(orc, rnd, k)
    inputs = [point_input(orc, P, fmt) for P in pts]
    edges = edge_scalars(rnd)
    ss = [b32(edges[i] if i < len(edges) else rnd.randrange(2**255)) for i in range(n)]
    idx = [rnd.randrange(k) for _ in range(n)] if indexed else None
    with Tables(eng, inputs, fmt) as t:
        got = t.mul(ss, idx, device)
    ts = idx or [0] * n
    assert got == [want(orc, s, pts[j], fmt) for s, j in zip(ss, ts)]
    assert got == mul_batch_each(eng, ss, [inputs[j] for j in ts], fmt)


@pytest.mark.parametrize("device", [False, True])
def test_unreduced_scalars_and_torsion(eng, orc, device):
    """Every edge scalar against random points, P + T for each 8-torsion T, the eight small-order points and the
    identity: the scalar is the integer it is, so a torsion component survives s = l."""
    rnd = random.Random(21 + device)
    tors = torsion_points(orc)
    prime = random_points(orc, rnd, 4)
    mixed = [orc.add(prime[0], T) for T in tors]
    pts = prime + mixed + [orc.identity()] + tors
    edges = edge_scalars(rnd)
    items = [(s, j) for s in edges for j in range(len(pts))]
    ss, ts = [b32(s) for s, _ in items], [j for _, j in items]
    for fmt in (COMPRESSED, EXTENDED):
        inputs = [point_input(orc, P, fmt) for P in pts]
        with Tables(eng, inputs, fmt) as t:
            got = t.mul(ss, ts, device)
        assert got == [want(orc, s, pts[j], fmt) for s, j in zip(ss, ts)]
        assert got == mul_batch_each(eng, ss, [inputs[j] for j in ts], fmt)
        for (s, j), g in zip(items, got):
            if s == L and 4 <= j < 4 + len(tors):                     # l (P + T) = l T = 5 T, not the identity
                assert g != b32(1) and g == orc.compress(orc.scalarmul(b32(5), tors[j - 4]))
    renc = [orc.ristretto_compress(P) for P in prime]
    items = [(s, j) for s in edges for j in range(len(prime))]
    ss, ts = [b32(s) for s, _ in items], [j for _, j in items]
    with Tables(eng, renc, RISTRETTO) as t:
        got = t.mul(ss, ts, device)
    assert got == [want(orc, s, prime[j], RISTRETTO) for s, j in zip(ss, ts)]
    assert got == mul_batch_each(eng, ss, [renc[j] for j in ts], RISTRETTO)


@pytest.mark.parametrize("fmt", [COMPRESSED, RISTRETTO])
@pytest.mark.parametrize("device", [False, True])
def test_clamped(eng, orc, fmt, device):
    rnd = random.Random(31 + fmt + device)
    pts = random_points(orc, rnd, 4)
    inputs = [point_input(orc, P, fmt) for P in pts]
    raw = [rnd.randbytes(32) for _ in range(300)] + [b"\xff" * 32, bytes(32)]
    idx = [rnd.randrange(4) for _ in raw]
    with Tables(eng, inputs, fmt) as t:
        one = t.mul(raw, None, device, clamped=True)
        many = t.mul(raw, idx, device, clamped=True)
    assert one == [want(orc, r, pts[0], fmt, True) for r in raw]
    assert many == [want(orc, r, pts[j], fmt, True) for r, j in zip(raw, idx)]
    if fmt == COMPRESSED:
        assert many == mul_batch_each(eng, raw, [inputs[j] for j in idx], fmt, clamped=True)


def test_ristretto_coset_invariance(eng, orc):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(41)
    tors = torsion_points(orc)
    four = [orc.identity(), tors[1], tors[3], tors[5]]          # the 4-torsion: orders 1, 4, 2, 4
    P = random_points(orc, rnd, 1)[0]
    ss = [b32(rnd.randrange(L)) for _ in range(50)] + [b32(L), b32(2**255 - 1)]
    reps = [orc.add(P, T) for T in four]
    encs = [orc.ristretto_compress(Q) for Q in reps]
    assert len(set(encs)) == 1
    outs, bases = [], []
    for e in encs:
        t = pkg.RistrettoBasepointTable.create(e, engine=eng)
        outs.append(t.mul_base_batch(ss))
        bases.append(t.basepoint())
        t.close()
    assert all(o == outs[0] for o in outs) and bases == [encs[0]] * 4
    assert outs[0] == [want(orc, s, P, RISTRETTO) for s in ss]
    # Edwards tables of the four representatives (extended limbs): different Edwards points, one Ristretto point
    k = len(reps)
    ext = b"".join(point_input(orc, Q, EXTENDED) for Q in reps)
    t = pkg.EdwardsBasepointTable((ext, k), engine=eng, fmt=EXTENDED)
    for j in range(k):
        got = t.mul_base_batch(ss, [j] * len(ss))
        assert [orc.ristretto_compress(orc.decompress(g)) for g in got] == outs[0]
        assert orc.ristretto_compress(orc.decompress(t.basepoint(j))) == encs[0]
    t.close()


@pytest.mark.parametrize("k", [2, 64, 1000])
@pytest.mark.parametrize("device", [False, True])
def test_many_tables(eng, orc, k, device):
    rnd = random.Random(51 + k + device)
    pts = random_points(orc, rnd, k)
    inputs = [orc.compress(P) for P in pts]
    n = 3000
    idx = [rnd.randrange(k) for _ in range(n)]
    idx[:40] = [0] * 20 + [k - 1] * 20                             # first, last, repeated
    idx[100:164] = [rnd.randrange(k)] * 64                          # one table for a whole warp and more
    ss = [b32(rnd.randrange(2**255)) for _ in range(n)]
    with Tables(eng, inputs, COMPRESSED) as t:
        got = t.mul(ss, idx, device)
    assert got == mul_batch_each(eng, ss, [inputs[j] for j in idx], COMPRESSED)
    for i in list(range(45)) + [rnd.randrange(n) for _ in range(30)]:
        assert got[i] == want(orc, ss[i], pts[idx[i]], COMPRESSED), i


@pytest.mark.parametrize("n", [PIECE - 1, PIECE + 1, 2 * PIECE + 3, 2 * PIECE + 5])
def test_piece_boundaries(eng, orc, n):
    import numpy as np
    rnd = random.Random(n)
    k = 5
    pts = random_points(orc, rnd, k)
    inputs = [orc.compress(P) for P in pts]
    raw = np.frombuffer(rnd.randbytes(32 * n), dtype=np.uint8).copy().reshape(n, 32)
    raw[:, 31] &= 0x7f
    ss = [bytes(r) for r in raw]
    idx = [rnd.randrange(k) for _ in range(n)]
    checks = sorted(i for i in {0, 1, PIECE - 1, PIECE, PIECE + 1, 2 * PIECE - 1, 2 * PIECE, n - 2, n - 1} | {rnd.randrange(n) for _ in range(10)} if i < n)
    with Tables(eng, inputs, COMPRESSED) as t:
        one = t.mul(ss)
        many = t.mul(ss, idx)
        many_dev = t.mul(ss, idx, device=True)
    rc, bc, _ = eng.mul_batch(b"".join(ss), n, inputs[0], 1, n)
    assert rc == 0 and one == split(bc)
    assert many == many_dev == mul_batch_each(eng, ss, [inputs[j] for j in idx], COMPRESSED)
    for i in checks:
        assert one[i] == want(orc, ss[i], pts[0], COMPRESSED), i
        assert many[i] == want(orc, ss[i], pts[idx[i]], COMPRESSED), i


def test_empty_batch(eng, orc):
    lib = eng.lib
    with Tables(eng, [orc.compress(orc.basepoint())] * 2, COMPRESSED) as t:
        assert lib.dalek_b200_basepoint_tables_mul(eng.h, t.h, None, None, 0, 0, None) == 0
        assert lib.dalek_b200_basepoint_tables_mul_dev(eng.h, t.h, None, None, 0, 0, None) == 0
        assert t.mul([]) == [] and t.mul([], []) == []


def test_basepoints(eng, orc):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(61)
    pts = random_points(orc, rnd, 5) + [orc.identity()] + torsion_points(orc)
    encs = [orc.compress(P) for P in pts]
    # non-canonical CompressedEdwardsY: y + p for the points with y < 19, and x = 0 with the sign bit set
    noncanon = []
    for y in range(19):
        for sign in (0, 1):
            e = bytearray(b32(y + P25519))
            e[31] |= sign << 7
            if orc.decompress(bytes(e)) is not None:
                noncanon.append(bytes(e))
    noncanon.append(b32(1 | 1 << 255))                               # the identity, "negative" x = 0
    assert len(noncanon) >= 3
    inputs = encs + noncanon
    with Tables(eng, inputs, COMPRESSED) as t:
        got = split(eng.basepoint_tables_basepoints(t.h))
    expect = [orc.compress(orc.decompress(e)) for e in inputs]
    assert got == expect and got[:len(encs)] == encs
    assert all(g != e for g, e in zip(got[len(encs):], noncanon))
    with Tables(eng, [point_input(orc, P, EXTENDED) for P in pts], EXTENDED) as t:
        assert split(eng.basepoint_tables_basepoints(t.h)) == encs
    renc = [orc.ristretto_compress(P) for P in pts[:5]]
    rt = pkg.RistrettoBasepointTable(renc, engine=eng)
    assert [rt.basepoint(i) for i in range(5)] == renc
    rt.close()


def test_errors(eng, eng2, orc):
    import curve25519_dalek_b200 as pkg
    lib, h = eng.lib, eng.h
    rnd = random.Random(71)
    pts = random_points(orc, rnd, 3)
    encs = b"".join(orc.compress(P) for P in pts)
    s, top = b32(5), b32(2**255 | 5)
    out = (C.c_uint8 * 64)()
    idx_ok, idx_bad = array.array("I", [2, 0]).tobytes(), array.array("I", [1, 3]).tobytes()
    with Tables(eng, split(encs), COMPRESSED) as t, Tables(eng, split(encs)[:1], COMPRESSED) as t1:
        mul = lib.dalek_b200_basepoint_tables_mul
        assert mul(h, t.h, top + s, None, 2, 0, out) == INVALID                 # bit 255 without the clamp flag
        assert mul(h, t.h, top + s, idx_ok, 2, 0, out) == INVALID
        assert mul(h, t.h, top + s, idx_ok, 2, 1, out) == 0                     # clamped: accepted
        assert mul(h, t.h, s + s, idx_bad, 2, 0, out) == INVALID                # index = k
        assert mul(h, t1.h, s + s, array.array("I", [0, 1]).tobytes(), 2, 0, out) == INVALID
        assert mul(h, t.h, s + s, idx_ok, 2, 2, out) == INVALID                 # unknown flag
        assert mul(h, t.h, None, None, 2, 0, out) == INVALID
        assert mul(h, t.h, s + s, None, 2, 0, None) == INVALID
        assert mul(h, None, s + s, None, 2, 0, out) == INVALID
        mdev = lib.dalek_b200_basepoint_tables_mul_dev
        d_top, d_s, d_out = dev(top + s), dev(s + s), dev(bytes(64))
        d_ok, d_bad = dev(idx_ok), dev(idx_bad)
        assert mdev(h, t.h, d_top.data_ptr(), None, 2, 0, d_out.data_ptr()) == INVALID
        assert mdev(h, t.h, d_top.data_ptr(), d_ok.data_ptr(), 2, 0, d_out.data_ptr()) == INVALID
        assert mdev(h, t.h, d_top.data_ptr(), d_ok.data_ptr(), 2, 1, d_out.data_ptr()) == 0
        assert mdev(h, t.h, d_s.data_ptr(), d_bad.data_ptr(), 2, 0, d_out.data_ptr()) == INVALID   # reported after the batch
        assert mdev(h, t1.h, d_s.data_ptr(), d_ok.data_ptr(), 2, 0, d_out.data_ptr()) == INVALID   # one table, index 2
        assert mdev(h, t1.h, d_s.data_ptr(), dev(bytes(8)).data_ptr(), 2, 0, d_out.data_ptr()) == 0
        # the engine still computes correctly after the reported errors
        assert t.mul([s, s], [2, 0], device=True) == [want(orc, s, pts[2], COMPRESSED), want(orc, s, pts[0], COMPRESSED)]
        # a handle of another context
        assert mul(eng2.h, t.h, s + s, None, 2, 0, out) == INVALID
        assert mdev(eng2.h, t.h, d_s.data_ptr(), None, 2, 0, d_out.data_ptr()) == INVALID
        assert lib.dalek_b200_basepoint_tables_basepoints(eng2.h, t.h, out) == INVALID
        assert lib.dalek_b200_basepoint_tables_len(t.h) == 3
    # new: an undecodable point, k = 0, bad formats
    new = lib.dalek_b200_basepoint_tables_new
    hh = C.c_void_p(1234)
    ok = (C.c_uint8 * 4)()
    bad = encs[:32] + b32(2) + encs[32:64] + b32(2)                             # y = 2 is not on the curve
    assert new(h, bad, COMPRESSED, 4, ok, C.byref(hh)) == DALEK_NONE
    assert hh.value is None and bytes(ok) == bytes([1, 0, 1, 0])
    assert new(h, bad, COMPRESSED, 4, None, C.byref(hh)) == DALEK_NONE and hh.value is None
    assert new(h, b32(2**255 - 1), RISTRETTO, 1, ok, C.byref(hh)) == DALEK_NONE and ok[0] == 0
    assert new(h, encs, COMPRESSED, 0, ok, C.byref(hh)) == INVALID and hh.value is None
    assert new(h, encs, 7, 3, ok, C.byref(hh)) == INVALID
    assert new(h, None, COMPRESSED, 3, ok, C.byref(hh)) == INVALID
    lib.dalek_b200_basepoint_tables_destroy(None)
    assert lib.dalek_b200_basepoint_tables_len(None) == 0
    # Python
    with pytest.raises(ValueError, match="point 1 "):
        pkg.EdwardsBasepointTable(split(bad), engine=eng)
    with pytest.raises(ValueError):
        pkg.EdwardsBasepointTable([], engine=eng)
    t = pkg.EdwardsBasepointTable(split(encs), engine=eng)
    with pytest.raises(ValueError):
        t.mul_base_batch([s, top])
    with pytest.raises(ValueError):
        t.mul_base_batch([s, s], [0, 3])
    with pytest.raises(ValueError):
        t.mul_base_batch([s, s], [0])
    t.close()
    t.close()


def test_reuse_and_concurrent_contexts(eng, eng2, orc):
    rnd = random.Random(81)
    tabs, expect = [], []
    for e in (eng, eng2):
        pts = random_points(orc, rnd, 8)
        ss = [b32(rnd.randrange(2**255)) for _ in range(20000)]
        idx = [rnd.randrange(8) for _ in ss]
        t = Tables(e, [orc.compress(P) for P in pts], COMPRESSED)
        tabs.append((t, ss, idx))
        expect.append(mul_batch_each(e, ss, [orc.compress(pts[j]) for j in idx], COMPRESSED))
    try:
        t, ss, idx = tabs[0]
        for _ in range(3):                                        # one handle, many calls, unchanged results
            assert t.mul(ss, idx) == expect[0]
            assert t.mul(ss[:100], idx[:100], device=True) == expect[0][:100]
            assert t.mul(ss[:7]) == t.mul(ss[:7], [0] * 7)
        results = [None, None]

        def run(j):
            tj, sj, ij = tabs[j]
            results[j] = [tj.mul(sj, ij) for _ in range(4)]

        threads = [threading.Thread(target=run, args=(j,)) for j in range(2)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        for j in range(2):
            assert all(r == expect[j] for r in results[j])
    finally:
        for t, _, _ in tabs:
            t.__exit__()


def test_python_wrappers(eng, orc):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(91)
    pts = random_points(orc, rnd, 3)
    encs = [orc.compress(P) for P in pts]
    t = pkg.EdwardsBasepointTable.create(encs[1], engine=eng)
    s = b32(rnd.randrange(L))
    assert len(t) == 1 and t.basepoint() == encs[1]
    assert t.mul_base_batch(s) == want(orc, s, pts[1], COMPRESSED)
    raw = rnd.randbytes(32)
    assert t.mul_base_clamped_batch([raw]) == [want(orc, raw, pts[1], COMPRESSED, True)]
    with pytest.raises(IndexError):
        t.basepoint(1)
    t.close()
    t = pkg.EdwardsBasepointTable(encs, engine=eng)
    ss = [b32(rnd.randrange(L)) for _ in range(6)]
    idx = [2, 0, 1, 1, 2, 0]
    assert len(t) == 3 and [t.basepoint(i) for i in range(3)] == encs
    assert t.mul_base_batch(ss, idx) == [want(orc, x, pts[j], COMPRESSED) for x, j in zip(ss, idx)]
    assert t.mul_base_batch(ss) == [want(orc, x, pts[0], COMPRESSED) for x in ss]
    assert t.mul_base_batch([]) == []
    del t
    renc = [orc.ristretto_compress(P) for P in pts]
    rt = pkg.RistrettoBasepointTable(renc, engine=eng)
    assert rt.mul_base_clamped_batch(raw, None) == want(orc, raw, pts[0], RISTRETTO, True)
    assert rt.mul_base_batch(ss, idx) == [want(orc, x, pts[j], RISTRETTO) for x, j in zip(ss, idx)]
    with pytest.raises(ValueError):
        pkg.RistrettoBasepointTable((b"", 0), engine=eng, fmt=EXTENDED)
    rt.close()


@pytest.mark.parametrize("k", [2, 1000])
@pytest.mark.parametrize("device", [False, True])
def test_grouped_and_ungrouped_agree(eng, orc, k, device):
    """The many-table path with its items grouped by table (option "bpt_group" 1, the default) and with every lane reading
    its own table give the same bytes, across the pieces of a host call and with runs of one table."""
    rnd = random.Random(101 + k + device)
    pts = random_points(orc, rnd, k)
    inputs = [orc.compress(P) for P in pts]
    n = 2 * PIECE + 7
    idx = [rnd.randrange(k) for _ in range(n)]
    idx[500:900] = [k - 1] * 400
    ss = [b32(rnd.randrange(2**255)) for _ in range(n)]
    assert eng.get_option("bpt_group") == 1
    with Tables(eng, inputs, COMPRESSED) as t:
        grouped = t.mul(ss, idx, device)
        eng.set_option("bpt_group", 0)
        try:
            plain = t.mul(ss, idx, device)
        finally:
            eng.set_option("bpt_group", 1)
        if device:                                                 # an index = k fails the grouped call, reads nothing outside
            d_s, d_bad, d_out = dev(b"".join(ss[:300])), dev(array.array("I", idx[:299] + [k]).tobytes()), dev(bytes(32 * 300))
            assert eng.lib.dalek_b200_basepoint_tables_mul_dev(eng.h, t.h, d_s.data_ptr(), d_bad.data_ptr(), 300, 0,
                                                               d_out.data_ptr()) == INVALID
    assert grouped == plain == mul_batch_each(eng, ss, [inputs[j] for j in idx], COMPRESSED)
    for i in [0, 500, 899, n - 1] + [rnd.randrange(n) for _ in range(10)]:
        assert grouped[i] == want(orc, ss[i], pts[idx[i]], COMPRESSED), i


def test_destroy_after_engine_close_and_extended_length(orc):
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    P = orc.basepoint()
    t = pkg.EdwardsBasepointTable([orc.compress(P)], engine=e)
    assert t.mul_base_batch(b32(7)) == orc.compress(orc.scalarmul(b32(7), P))
    e.close()
    t.close()                                                      # the handle does not use the closed context
    ext = point_input(orc, P, EXTENDED)
    with pytest.raises(ValueError):
        pkg.EdwardsBasepointTable((ext, 2), engine=e, fmt=EXTENDED)
