"""CPU checks of the batched Scalar arithmetic: the host build of sc_sub, sc_div_by_2, sc_is_canonical and sc_invert
(csrc/sc.cuh) against Python integers and the C oracle; the fold's chunk plan (csrc/ps_plan.h) against a Python model;
the scalar known answers of tests/golden/scalar_ops.json against Python integers; and the SASS / resource usage of the
new kernels in the built library."""
import ctypes as C
import json
import os
import random
import re
import subprocess
import sys

import pytest

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")
L = 2**252 + 27742317777372353535851937790883648493
CHUNK, PIECE = 1024, 1 << 18           # SF_CHUNK and SF_PIECE of scalars.cu

sys.path.insert(0, GOLDEN)
import make_scalar_golden  # noqa: E402

EDGES = [0, 1, 2, L - 1, (L - 1) // 2, (L + 1) // 2, 2**252 - 1, 2**252, L, 2**255 - 1, 2**256 - 1]
CANONICAL_EDGES = [x for x in EDGES if x < L]


@pytest.fixture(scope="module")
def sc():
    src = os.path.join(ROOT, "tests", "host", "scalar_ops_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libscalaropshost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("sc.cuh", "constants.cuh", "fe.cuh", "ps_plan.h")]
    if not os.access(os.path.dirname(so), os.W_OK):
        import tempfile
        so = os.path.join(tempfile.mkdtemp(prefix="scalaropshost_"), "libscalaropshost.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    for f in ("h_sc_sub", "h_sc_div_by_2", "h_sc_invert", "h_sc_is_canonical"):
        getattr(lib, f).restype = None
    lib.h_plan.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.h_pieces.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.h_pieces.restype = C.c_size_t
    lib.h_offsets_ok.argtypes = [C.c_void_p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


def _buf(vals):
    return (C.c_uint8 * max(1, 32 * len(vals))).from_buffer_copy(b"".join(v.to_bytes(32, "little") for v in vals) or b"\0")


def _ints(buf, n):
    raw = bytes(buf)
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(n)]


def run2(lib, name, a, b):
    o = (C.c_uint8 * (32 * len(a)))()
    getattr(lib, name)(o, _buf(a), _buf(b), C.c_size_t(len(a)))
    return _ints(o, len(a))


def run1(lib, name, a):
    o = (C.c_uint8 * (32 * len(a)))()
    getattr(lib, name)(o, _buf(a), C.c_size_t(len(a)))
    return _ints(o, len(a))


def b32(x):
    return x.to_bytes(32, "little")


def test_sc_sub_against_integers_and_oracle(sc, orc):
    rnd = random.Random(11)
    pairs = [(x, y) for x in CANONICAL_EDGES for y in CANONICAL_EDGES]
    pairs += [(rnd.randrange(L), rnd.randrange(L)) for _ in range(50000)]
    a, b = [p[0] for p in pairs], [p[1] for p in pairs]
    got = run2(sc, "h_sc_sub", a, b)
    assert got == [(x - y) % L for x, y in pairs]
    for (x, y), g in list(zip(pairs, got))[:len(CANONICAL_EDGES) ** 2 + 500]:
        assert b32(g) == orc.sc_op2("scalar_sub", b32(x), b32(y)), (x, y)


def test_sc_div_by_2(sc):
    rnd = random.Random(12)
    xs = CANONICAL_EDGES + [(-i) % L for i in range(64)] + list(range(64)) + [rnd.randrange(L) for _ in range(50000)]
    got = run1(sc, "h_sc_div_by_2", xs)
    inv2 = (L + 1) // 2
    assert got == [x * inv2 % L for x in xs]
    assert all(2 * g % L == x for g, x in zip(got, xs))


def test_sc_is_canonical(sc, orc):
    rnd = random.Random(13)
    xs = EDGES + [L + i for i in range(-3, 4)] + [rnd.randrange(2**256) for _ in range(20000)] + \
        [rnd.randrange(L) for _ in range(20000)] + [rnd.randrange(L, 2**253) for _ in range(2000)]
    o = (C.c_uint8 * len(xs))()
    sc.h_sc_is_canonical(o, _buf(xs), C.c_size_t(len(xs)))
    assert list(o) == [int(x < L) for x in xs]
    for x in xs[:400]:
        assert bool(o[xs.index(x)]) == orc.scalar_is_canonical(b32(x))


def test_sc_invert_against_integers_and_oracle(sc, orc):
    rnd = random.Random(14)
    xs = CANONICAL_EDGES + [rnd.randrange(L) for _ in range(300)]
    got = run1(sc, "h_sc_invert", xs)
    assert got == [pow(x, L - 2, L) for x in xs]
    assert got[0] == 0                                               # invert(0) = 0
    for x, g in zip(xs[:60], got):
        assert b32(g) == orc.sc_op1("scalar_invert", b32(x))


def test_golden_fixture_is_self_consistent():
    with open(os.path.join(GOLDEN, "scalar_ops.json")) as f:
        g = json.load(f)
    make_scalar_golden.check(g)
    with open(os.path.join(GOLDEN, "kat.json")) as f:
        kat = json.load(f)["scalar"]
    for name in ("X", "XINV", "Y", "X_TIMES_Y"):
        assert g[name]["hex"] == kat[name]["hex"]


def test_golden_against_host_build(sc):
    with open(os.path.join(GOLDEN, "scalar_ops.json")) as f:
        g = json.load(f)
    n = lambda h: int.from_bytes(bytes.fromhex(h), "little")   # noqa: E731
    assert run1(sc, "h_sc_invert", [n(g["invert"]["s"])]) == [n(g["invert"]["inv"])]
    cases = g["div_by_2"]["cases"]
    assert run1(sc, "h_sc_div_by_2", [n(c["s"]) for c in cases]) == [n(c["half"]) for c in cases]
    enc = [n(c["bytes"]) for c in g["canonical_decoding"]["cases"]]
    o = (C.c_uint8 * len(enc))()
    sc.h_sc_is_canonical(o, _buf(enc), C.c_size_t(len(enc)))
    assert [bool(v) for v in o] == [c["canonical"] for c in g["canonical_decoding"]["cases"]]


# ---- the chunk plan of the fold (ps_plan.h, shared with the point sum) ---------------------------------------------------
def model_plan(offsets, chunk):
    start, base = [], []
    for lo, hi in zip(offsets[:-1], offsets[1:]):
        base.append(len(start))
        start.extend(range(lo, hi, chunk))
    base.append(len(start))
    start.append(offsets[-1])
    lens = [b - a for a, b in zip(start[:-1], start[1:])]
    per_seg = [b - a for a, b in zip(base[:-1], base[1:])]
    return start, base, max(lens, default=0), max(per_seg, default=0)


def model_pieces(start, piece):
    cuts = [0]
    for c in range(len(start) - 1):
        if start[c + 1] - start[cuts[-1]] > piece:
            cuts.append(c)
    if cuts[-1] != len(start) - 1:
        cuts.append(len(start) - 1)
    return cuts


SHAPES = {
    "empty": [0], "empties": [0, 0, 0], "singletons": [1] * 300, "chunk_edges": [CHUNK - 1, CHUNK, CHUNK + 1],
    "across_pieces": [PIECE - 3, 2 * CHUNK + 5, PIECE + 1, 0, 7], "one_long": [(1 << 22)], "many_16": [16] * 4096,
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_fold_plan_against_model(sc, shape):
    sizes = SHAPES[shape]
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    m = len(sizes)
    assert sc.h_offsets_ok((C.c_uint64 * (m + 1))(*offs), m) == 1
    levels = 0
    while True:
        n_max = sum((s + CHUNK - 1) // CHUNK for s in sizes) + 1
        start, base, info = (C.c_uint32 * n_max)(), (C.c_uint32 * (m + 1))(), (C.c_uint32 * 3)()
        sc.h_plan((C.c_uint64 * (m + 1))(*offs), m, CHUNK, start, base, info)
        start = list(start)[:info[0] + 1]
        assert (start, list(base), info[1], info[2]) == model_plan(offs, CHUNK)
        nch = len(start) - 1
        cuts = (C.c_uint32 * (nch + 2))()
        k = sc.h_pieces((C.c_uint32 * len(start))(*start), nch, PIECE, cuts)
        assert list(cuts)[:k] == model_pieces(start, PIECE)
        levels += 1
        if info[2] <= 1:
            break
        offs, sizes = list(base), [b - a for a, b in zip(list(base)[:-1], list(base)[1:])]
    assert levels <= 3                   # 2^22 scalars: 4096 chunks, 4 partials, 1


def test_fold_offsets_rule(sc):
    def ok(offs):
        return sc.h_offsets_ok((C.c_uint64 * len(offs))(*offs), len(offs) - 1)
    assert ok([0, 3, 3, 9]) == 1
    assert ok([1, 3]) == 0 and ok([0, 5, 4]) == 0 and ok([0, 2**31]) == 0 and ok([0, 2**31 - 1]) == 1


# ---- SASS of the kernels -----------------------------------------------------------------------------------------------
# kernel -> (mangled name prefix, instantiations, bytes of stack frame as DESIGN.md section 9 records them: CUDA 12.9,
# sm_90a).  The 32 bytes of the per-item inversion hold the public exponent l - 2, indexed by the bit position (as in
# k_scalar_invert_groups), never a scalar.
KERNELS = {"k_scalar_binary": ("15k_scalar_binaryILi", 3, 0), "k_scalar_unary": ("14k_scalar_unaryILi", 3, 32),
           "k_scalar_from_bytes": ("19k_scalar_from_bytesILi", 2, 0), "k_scalar_hash_bytes": ("19k_scalar_hash_bytes", 1, 0),
           "k_scalar_fold_chunks": ("20k_scalar_fold_chunksILi", 2, 0),
           "k_scalar_fold_finish": ("20k_scalar_fold_finishILi", 2, 0)}


def _need_lib():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")


def _function_sections(text, name):
    blocks, cur = [], None
    for line in text.splitlines():
        m = re.search(r"Function\s*:\s*(\S+)", line)
        if m:
            cur = [] if name in m.group(1) else None
            if cur is not None:
                blocks.append(cur)
        if cur is not None:
            cur.append(line)
    return ["\n".join(b) for b in blocks]


@pytest.fixture(scope="module")
def sass():
    _need_lib()
    return subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_kernel_sass_has_no_indirect_branch(sass, kernel):
    name, count, _ = KERNELS[kernel]
    blocks = _function_sections(sass, name)
    assert len(blocks) == count, kernel
    for block in blocks:
        assert not re.search(r"\b(BRX|JMX)\b", block)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_kernel_resource_usage(kernel):
    _need_lib()
    name, count, stack_max = KERNELS[kernel]
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    idx = [i for i, l in enumerate(lines) if re.search(r"Function\s+\S*" + name, l)]
    assert len(idx) == count, kernel
    for i in idx:
        usage = lines[i + 1]
        stack, local = re.search(r"\bSTACK:(\d+)\b", usage), re.search(r"\bLOCAL:(\d+)\b", usage)
        assert stack and local, usage
        assert int(local.group(1)) == 0, usage
        assert int(stack.group(1)) <= stack_max, usage
