"""The batched Scalar arithmetic on the GPU (csrc/scalars.cu) against Python integers mod l and the C oracle: Add / Sub /
Mul / Neg / invert / div_by_2 at piece boundaries, with broadcast on either side, on host and device buffers and in
place; the rejection of non-canonical inputs at every position for every op; the byte constructors and hash_from_bytes;
segmented Sum / Product; Schnorr signing and Shamir reconstruction through engine calls only; and the argument checks."""
import ctypes as C
import hashlib
import json
import os
import random

import numpy as np
import pytest

import curve25519_dalek_b200 as pkg
import oracle_lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = 2**252 + 27742317777372353535851937790883648493
INV2 = (L + 1) // 2
PIECE = 1 << 16                       # SC_PIECE of scalars.cu
FOLD_PIECE = 1 << 18                  # SF_PIECE
SIZES = [1, PIECE - 1, PIECE + 1, 3 * PIECE + 5]
EDGES = [0, 1, 2, L - 1, (L - 1) // 2, (L + 1) // 2, 2**252 - 1, 2**252]
BAD = [L, 2**255 - 1, 2**255 + 7]      # >= l, the largest unreduced, bit 255 set
E_INVALID = -1
BINARY = {"add": lambda x, y: (x + y) % L, "sub": lambda x, y: (x - y) % L, "mul": lambda x, y: x * y % L}
UNARY = {"neg": lambda x: (-x) % L, "invert": lambda x: pow(x, L - 2, L), "div_by_2": lambda x: x * INV2 % L}
ORACLE = {"add": "scalar_add", "sub": "scalar_sub", "mul": "scalar_mul", "neg": "scalar_neg", "invert": "scalar_invert"}


def b32(x):
    return x.to_bytes(32, "little")


def enc(xs):
    return b"".join(b32(x) for x in xs)


def dec(raw, n=None):
    raw = bytes(raw.cpu().numpy().tobytes()) if hasattr(raw, "cpu") else bytes(raw)
    n = len(raw) // 32 if n is None else n
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(n)]


def dev(raw):
    import torch
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()


@pytest.fixture(scope="module")
def eng():
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "scalar_ops.json")) as f:
        return json.load(f)


class Pool:
    """Item i of a batch is pool[(k i + c) % P]: large batches with cheap expected values (the inverses are cached)."""

    def __init__(self, seed, size=4093):
        rnd = random.Random(seed)
        self.v = EDGES + [rnd.randrange(L) for _ in range(size - len(EDGES))]
        self.inv = {}

    def items(self, n, k=1, c=0):
        return [self.v[(k * i + c) % len(self.v)] for i in range(n)]

    def unary(self, op, x):
        if op == "invert":
            if x not in self.inv:
                self.inv[x] = UNARY["invert"](x)
            return self.inv[x]
        return UNARY[op](x)


@pytest.fixture(scope="module")
def pool():
    return Pool(7)


# ---- element-wise ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("op", sorted(BINARY))
def test_binary_host(eng, orc, pool, op, n):
    a, b = pool.items(n), pool.items(n, 3, 1)
    got = dec(eng.scalar_binary_batch(op, enc(a), n, enc(b), n, n), n)
    assert got == [BINARY[op](x, y) for x, y in zip(a, b)]
    for x, y, g in list(zip(a, b, got))[:24]:
        assert b32(g) == orc.sc_op2(ORACLE[op], b32(x), b32(y))


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("op", sorted(UNARY))
def test_unary_host(eng, orc, pool, op, n):
    a = pool.items(n, 5, 2)
    got = dec(eng.scalar_unary_batch(op, enc(a), n), n)
    assert got == [pool.unary(op, x) for x in a]
    if op in ORACLE:
        for x, g in list(zip(a, got))[:24]:
            assert b32(g) == orc.sc_op1(ORACLE[op], b32(x))


@pytest.mark.parametrize("side", ["a", "b"])
@pytest.mark.parametrize("op", sorted(BINARY))
def test_binary_broadcast_host_and_device(eng, pool, op, side):
    n = PIECE + 1
    one, many = pool.v[9], pool.items(n, 11, 4)
    a, na, b, nb = (b32(one), 1, enc(many), n) if side == "a" else (enc(many), n, b32(one), 1)
    want = [BINARY[op](one, y) if side == "a" else BINARY[op](y, one) for y in many]
    assert dec(eng.scalar_binary_batch(op, a, na, b, nb, n), n) == want
    assert dec(eng.scalar_binary_batch(op, dev(a), na, dev(b), nb, n, device_ptrs=True), n) == want


@pytest.mark.parametrize("op", sorted(BINARY))
def test_binary_device_and_in_place(eng, pool, op):
    n = 3 * PIECE + 5
    a, b = pool.items(n, 13, 3), pool.items(n, 17, 5)
    want = [BINARY[op](x, y) for x, y in zip(a, b)]
    da, db = dev(enc(a)), dev(enc(b))
    assert dec(eng.scalar_binary_batch(op, da, n, db, n, n, device_ptrs=True), n) == want
    eng.scalar_binary_batch(op, da, n, db, n, n, device_ptrs=True, out=da)        # out = a
    assert dec(da, n) == want
    da = dev(enc(a))
    eng.scalar_binary_batch(op, da, n, db, n, n, device_ptrs=True, out=db)        # out = b
    assert dec(db, n) == want


@pytest.mark.parametrize("op", sorted(UNARY))
def test_unary_device_and_in_place(eng, pool, op):
    n = PIECE + 1
    a = pool.items(n, 19, 6)
    want = [pool.unary(op, x) for x in a]
    da = dev(enc(a))
    assert dec(eng.scalar_unary_batch(op, da, n, device_ptrs=True), n) == want
    eng.scalar_unary_batch(op, da, n, device_ptrs=True, out=da)
    assert dec(da, n) == want


def test_chains_stay_on_the_device(eng, pool):
    """((a + b) * c - a) / 2, negated and inverted, in place on one device buffer."""
    n = PIECE + 3
    a, b, c = pool.items(n, 1, 0), pool.items(n, 7, 1), pool.items(n, 23, 2)
    da, db, dc, acc = dev(enc(a)), dev(enc(b)), dev(enc(c)), dev(enc(a))
    eng.scalar_binary_batch("add", acc, n, db, n, n, device_ptrs=True, out=acc)
    eng.scalar_binary_batch("mul", acc, n, dc, n, n, device_ptrs=True, out=acc)
    eng.scalar_binary_batch("sub", acc, n, da, n, n, device_ptrs=True, out=acc)
    for op in ("div_by_2", "neg", "invert"):
        eng.scalar_unary_batch(op, acc, n, device_ptrs=True, out=acc)
    want = [pow((-(((x + y) * z - x) * INV2)) % L, L - 2, L) for x, y, z in zip(a, b, c)]
    assert dec(acc, n) == want


# ---- non-canonical inputs --------------------------------------------------------------------------------------------
REJECT_OPS = ["add:a", "add:b", "sub:a", "sub:b", "mul:a", "mul:b", "neg", "invert", "div_by_2", "sum", "product"]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("kind", ["host", "device"])
@pytest.mark.parametrize("op", REJECT_OPS)
def test_non_canonical_input_is_rejected(eng, pool, op, kind, where):
    n = PIECE + 1
    good = pool.items(n, 29, 8)
    at = {"first": 0, "middle": n // 2, "last": n - 1}[where]
    name, _, operand = op.partition(":")
    wrap = dev if kind == "device" else (lambda raw: raw)
    offs = np.array([0, n // 3, n], dtype=np.uint64)
    for v in BAD:
        items = list(good)
        items[at] = v
        bad = enc(items)
        with pytest.raises(pkg.EngineError, match="not canonical"):
            if name in BINARY:
                a, b = (bad, enc(good)) if operand == "a" else (enc(good), bad)
                eng.scalar_binary_batch(name, wrap(a), n, wrap(b), n, n, device_ptrs=kind == "device")
            elif name in UNARY:
                eng.scalar_unary_batch(name, wrap(bad), n, device_ptrs=kind == "device")
            else:
                eng.scalar_fold_batch(name, wrap(bad), wrap(offs.tobytes()) if kind == "device" else offs, 2,
                                      device_ptrs=kind == "device")
    # the engine is still good afterwards
    assert dec(eng.scalar_unary_batch("neg", enc(good[:5]), 5)) == [(-x) % L for x in good[:5]]


def test_non_canonical_broadcast_operand_is_rejected(eng, pool):
    n = PIECE + 1
    for v in BAD:
        with pytest.raises(pkg.EngineError, match="not canonical"):
            eng.scalar_binary_batch("mul", b32(v), 1, enc(pool.items(n)), n, n)
        with pytest.raises(pkg.EngineError, match="not canonical"):
            eng.scalar_binary_batch("add", dev(enc(pool.items(n))), n, dev(b32(v)), 1, n, device_ptrs=True)


# ---- constructors, invert, hashing -----------------------------------------------------------------------------------
def test_from_bytes_mod_order(eng, orc):
    rnd = random.Random(21)
    xs = EDGES + BAD + [2**256 - 1, 2 * L, 8 * L - 1] + [rnd.randrange(2**256) for _ in range(PIECE + 40)]
    got = pkg.Scalar.from_bytes_mod_order_batch([b32(x) for x in xs], engine=eng)
    assert [int.from_bytes(g, "little") for g in got] == [x % L for x in xs]
    for x in xs[:40]:
        assert orc.sc_op1("scalar_reduce", b32(x)) == b32(x % L)
    rc, _, ok = eng.scalar_from_bytes_batch(enc(xs), len(xs))
    assert rc == 0 and ok == b"\1" * len(xs)


def test_from_canonical_bytes(eng, orc, golden):
    rnd = random.Random(22)
    xs = EDGES + BAD + [L + 1, 2**256 - 1] + [rnd.randrange(2**256) for _ in range(PIECE + 40)]
    rc, raw, ok = eng.scalar_from_bytes_batch(enc(xs), len(xs), canonical=True)
    assert rc == 1
    assert list(ok) == [int(x < L) for x in xs]
    assert dec(raw, len(xs)) == [x if x < L else 0 for x in xs]
    assert [bool(o) for o in ok[:60]] == [orc.scalar_is_canonical(b32(x)) for x in xs[:60]]
    rc, _, ok = eng.scalar_from_bytes_batch(enc(EDGES), len(EDGES), canonical=True)
    assert rc == 0 and ok == b"\1" * len(EDGES)
    cases = golden["canonical_decoding"]["cases"]
    got = pkg.Scalar.from_canonical_bytes_batch([bytes.fromhex(c["bytes"]) for c in cases], engine=eng)
    assert [g is not None for g in got] == [c["canonical"] for c in cases]
    assert got[0] == bytes.fromhex(cases[0]["bytes"])


def test_invert_each(eng, pool, golden):
    assert pkg.Scalar.invert_each(bytes(32), engine=eng) == bytes(32)                # invert(0) = 0
    xs = [x for x in pool.v[:500] if x]
    each = pkg.Scalar.invert_each([b32(x) for x in xs], engine=eng)
    inv, prod = pkg.Scalar.invert_batch_alloc([b32(x) for x in xs], engine=eng)
    assert each == inv
    p = 1
    for x in xs:
        p = p * pow(x, L - 2, L) % L
    assert prod == b32(p)
    assert pkg.Scalar.invert_each(bytes.fromhex(golden["invert"]["s"]), engine=eng).hex() == golden["invert"]["inv"]
    with pytest.raises(pkg.EngineError):
        pkg.Scalar.invert_batch_alloc([b32(3), bytes(32)], engine=eng)


def test_golden_neg_div_mul(eng, golden):
    g = golden
    x = bytes.fromhex(g["X"]["hex"])
    assert pkg.Scalar.neg_batch(pkg.Scalar.neg_batch(x, engine=eng), engine=eng) == x
    assert pkg.Scalar.neg_batch(x, engine=eng).hex() == g["neg_twice_is_identity"]["neg"]
    assert pkg.Scalar.mul_batch(x, bytes.fromhex(g["Y"]["hex"]), engine=eng).hex() == g["X_TIMES_Y"]["hex"]
    cases = g["div_by_2"]["cases"]
    halves = pkg.Scalar.div_by_2_batch([bytes.fromhex(c["s"]) for c in cases], engine=eng)
    assert [h.hex() for h in halves] == [c["half"] for c in cases]
    assert pkg.Scalar.add_batch(halves, halves, engine=eng) == [bytes.fromhex(c["s"]) for c in cases]
    assert pkg.Scalar.neg_batch(bytes(32), engine=eng) == bytes(32)


def test_hash_from_bytes(eng, golden):
    rnd = random.Random(23)
    msgs = [rnd.randbytes(k) for k in (0, 1, 111, 112, 127, 128, 239, 240, 300)]
    msgs += [rnd.randbytes(rnd.randrange(200)) for _ in range(PIECE + 7)]
    got = pkg.Scalar.hash_from_bytes_batch(msgs, engine=eng)
    assert got == [b32(int.from_bytes(hashlib.sha512(m).digest(), "little") % L) for m in msgs]
    fh = golden["from_hash"]
    assert pkg.Scalar.hash_from_bytes_batch([bytes.fromhex(fh["message"])], engine=eng)[0].hex() == fh["scalar"]
    assert pkg.Scalar.hash_from_bytes_batch([], engine=eng) == []


# ---- Sum / Product ---------------------------------------------------------------------------------------------------
def fold_want(op, items):
    if op == "sum":
        return sum(items) % L
    p = 1
    for x in items:
        p = p * x % L
    return p


FOLD_SHAPES = {
    "empty_and_singletons": [0, 1, 0, 0, 1, 1, 0],
    "chunk_edges": [1023, 1024, 1025, 2047, 2048, 2049],
    "across_pieces": [FOLD_PIECE - 3, 5000, FOLD_PIECE + 1, 0, 7, 3 * 1024 + 1],
    "many_16": [16] * (1 << 16),
    "one_long": [1 << 22],
}


@pytest.mark.parametrize("kind", ["host", "device"])
@pytest.mark.parametrize("op", ["sum", "product"])
@pytest.mark.parametrize("shape", sorted(FOLD_SHAPES))
def test_fold(eng, pool, shape, op, kind):
    sizes = FOLD_SHAPES[shape]
    offs = np.zeros(len(sizes) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(sizes)
    total = int(offs[-1])
    items = pool.items(total, 31, 9)
    flat = enc(items)
    if kind == "host":
        raw = eng.scalar_fold_batch(op, flat, offs, len(sizes))
    else:
        raw = eng.scalar_fold_batch(op, dev(flat), dev(offs.tobytes()), len(sizes), device_ptrs=True)
    want = [fold_want(op, items[int(a):int(b)]) for a, b in zip(offs[:-1], offs[1:])]
    assert dec(raw, len(sizes)) == want


def test_fold_golden_and_wrappers(eng, golden):
    for c in golden["impl_sum"]["cases"]:
        assert pkg.Scalar.sum([bytes.fromhex(v) for v in c["items"]], engine=eng).hex() == c["sum"]
    for c in golden["impl_product"]["cases"]:
        assert pkg.Scalar.product([bytes.fromhex(v) for v in c["items"]], engine=eng).hex() == c["product"]
    lists = [[bytes.fromhex(v) for v in c["items"]] for c in golden["impl_sum"]["cases"]]
    assert [s.hex() for s in pkg.Scalar.sum_batch(lists, engine=eng)] == [c["sum"] for c in golden["impl_sum"]["cases"]]
    lists = [[bytes.fromhex(v) for v in c["items"]] for c in golden["impl_product"]["cases"]]
    assert [s.hex() for s in pkg.Scalar.product_batch(lists, engine=eng)] == [c["product"] for c in golden["impl_product"]["cases"]]
    assert pkg.Scalar.sum_batch([], engine=eng) == []


# ---- end to end -------------------------------------------------------------------------------------------------------
def test_schnorr_sign_and_verify(eng):
    """k = hash_from_bytes(R || A || M), s = r + k a; R = [s]B - [k]A by the vartime double-base batch."""
    rnd = random.Random(24)
    n = 200
    S = pkg.Scalar
    a = [b32(rnd.randrange(L)) for _ in range(n)]
    r = [b32(rnd.randrange(L)) for _ in range(n)]
    msgs = [rnd.randbytes(rnd.randrange(100)) for _ in range(n)]
    A = pkg.EdwardsPoint.mul_base_batch(a, engine=eng)
    R = pkg.EdwardsPoint.mul_base_batch(r, engine=eng)
    k = S.hash_from_bytes_batch([R[i] + A[i] + msgs[i] for i in range(n)], engine=eng)
    s = S.add_batch(r, S.mul_batch(k, a, engine=eng), engine=eng)
    assert pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch(S.neg_batch(k, engine=eng), A, s, engine=eng) == R
    bad = list(s)
    bad[17] = S.add_batch(bad[17], b32(1), engine=eng)
    got = pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch(S.neg_batch(k, engine=eng), A, bad, engine=eng)
    assert [g == w for g, w in zip(got, R)] == [i != 17 for i in range(n)]


def test_shamir_reconstruction(eng):
    """Shares y_i = f(x_i) of f of degree t - 1; f(0) from t shares by Lagrange coefficients
    lambda_i = prod_j x_j / (x_j - x_i), built with sub, product_batch, invert_each, mul and sum."""
    rnd = random.Random(25)
    S = pkg.Scalar
    t, nshares = 7, 12
    coef = [rnd.randrange(L) for _ in range(t)]
    xs = [rnd.randrange(1, L) for _ in range(nshares)]
    ys = [sum(c * pow(x, e, L) for e, c in enumerate(coef)) % L for x in xs]
    pick = rnd.sample(range(nshares), t)
    num_lists, den_lists = [], []
    for i in pick:
        others = [j for j in pick if j != i]
        num_lists.append([b32(xs[j]) for j in others])
        den_lists.append(S.sub_batch([b32(xs[j]) for j in others], b32(xs[i]), engine=eng))
    lam = S.mul_batch(S.product_batch(num_lists, engine=eng),
                      S.invert_each(S.product_batch(den_lists, engine=eng), engine=eng), engine=eng)
    secret = S.sum(S.mul_batch(lam, [b32(ys[i]) for i in pick], engine=eng), engine=eng)
    assert secret == b32(coef[0])


# ---- argument checks -------------------------------------------------------------------------------------------------
def test_argument_checks(eng):
    lib, h = eng.lib, eng.h
    one = (C.c_uint8 * 64)()
    out = (C.c_uint8 * 64)()
    offs = (C.c_uint64 * 3)(0, 1, 2)
    huge = 1 << 62
    assert lib.dalek_b200_scalar_binary_batch(h, 3, one, 1, one, 1, 1, out) == E_INVALID          # bad op
    assert lib.dalek_b200_scalar_binary_batch(h, -1, one, 1, one, 1, 1, out) == E_INVALID
    assert lib.dalek_b200_scalar_unary_batch(h, 3, one, 1, out) == E_INVALID
    assert lib.dalek_b200_scalar_fold_batch(h, 2, one, offs, 2, out) == E_INVALID
    assert lib.dalek_b200_scalar_from_bytes_batch(h, one, 1, 2, out, None) == E_INVALID          # bad mode
    assert lib.dalek_b200_scalar_binary_batch(h, 0, one, 2, one, 1, 3, out) == E_INVALID         # n_a not 1 or n
    assert lib.dalek_b200_scalar_binary_batch(h, 0, None, 1, one, 1, 1, out) == E_INVALID        # NULL buffers
    assert lib.dalek_b200_scalar_binary_batch(h, 0, one, 1, one, 1, 1, None) == E_INVALID
    assert lib.dalek_b200_scalar_unary_batch(h, 0, None, 1, out) == E_INVALID
    assert lib.dalek_b200_scalar_from_bytes_batch(h, one, 1, 0, None, None) == E_INVALID
    assert lib.dalek_b200_scalar_hash_from_bytes_batch(h, one, None, 1, out) == E_INVALID
    assert lib.dalek_b200_scalar_fold_batch(h, 0, None, offs, 2, out) == E_INVALID
    assert lib.dalek_b200_scalar_fold_batch(h, 0, one, None, 2, out) == E_INVALID
    assert lib.dalek_b200_scalar_binary_batch(h, 0, one, huge, one, huge, huge, out) == E_INVALID  # sizes that overflow
    assert lib.dalek_b200_scalar_unary_batch(h, 0, one, huge, out) == E_INVALID
    assert lib.dalek_b200_scalar_from_bytes_batch(h, one, huge, 0, out, None) == E_INVALID
    assert lib.dalek_b200_scalar_hash_from_bytes_batch(h, one, offs, huge, out) == E_INVALID
    assert lib.dalek_b200_scalar_fold_batch(h, 0, one, offs, huge, out) == E_INVALID
    for bad in ((1, 2), (0, 2, 1), (0, 1 << 31)):                                                 # bad offsets
        o = (C.c_uint64 * len(bad))(*bad)
        assert lib.dalek_b200_scalar_fold_batch(h, 0, one, o, len(bad) - 1, out) == E_INVALID
    flat = (C.c_uint8 * 8)()
    assert lib.dalek_b200_scalar_hash_from_bytes_batch(h, flat, (C.c_uint64 * 3)(0, 5, 4), 2, out) == E_INVALID
    # n = 0 / m = 0: successful no-ops, NULL buffers allowed
    assert lib.dalek_b200_scalar_binary_batch(h, 0, None, 0, None, 0, 0, None) == 0
    assert lib.dalek_b200_scalar_unary_batch_dev(h, 1, None, 0, None) == 0
    assert lib.dalek_b200_scalar_fold_batch(h, 1, None, None, 0, None) == 0
    assert lib.dalek_b200_scalar_from_bytes_batch(h, None, 0, 1, None, None) == 0
    assert lib.dalek_b200_scalar_hash_from_bytes_batch(h, None, None, 0, None) == 0
    # every call sets last_call_ms; an empty segment list is fine with a NULL scalar buffer
    assert lib.dalek_b200_scalar_fold_batch(h, 1, None, (C.c_uint64 * 3)(0, 0, 0), 2, out) == 0
    assert bytes(out)[:64] == b32(1) * 2
    eng.scalar_binary_batch("mul", enc([3] * 1000), 1000, enc([5] * 1000), 1000, 1000)
    assert eng.last_call_ms() > 0
