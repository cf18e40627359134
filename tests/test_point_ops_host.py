"""Host build of the group operations (csrc/point_ops.cuh) with the fe / fe64 limb-bound and scale assertions on, against
the C oracle; the segmented sum's chunk plan against a Python model; and the SASS / resource usage of the new kernels in
the built library.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

import oracle_lib
import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
L = pyref.L
PRIME = 2**255 - 19
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
ADD, SUB, NEG, DOUBLE, COFACTOR = range(5)
ENC_EDWARDS, ENC_RISTRETTO, ENC_LIMBS = 0, 1, 2
CHUNK, PIECE = 1024, 1 << 16           # PS_CHUNK and PS_PIECE of point_ops.cu


@pytest.fixture(scope="module")
def host():
    src = os.path.join(ROOT, "tests", "host", "point_ops_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libpointopshost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("point_ops.cuh", "ge64.cuh", "ge.cuh", "fe64.cuh", "fe.cuh", "constants.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_op.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
    lib.h_eq.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    lib.h_sum.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
    lib.h_plan.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.h_pieces.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.h_pieces.restype = C.c_size_t
    return lib


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def torsion():
    with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json")) as f:
        return json.load(f)["EIGHT_TORSION"]


def b32(x):
    return x.to_bytes(32, "little")


def limbs_bytes(limbs):
    return b"".join(int(v).to_bytes(8, "little") for v in limbs)


def op(host, o, a, b=None, fmt=COMPRESSED, enc=ENC_EDWARDS):
    out = (C.c_uint8 * 160)()
    ok = host.h_op(out, bytes(a), bytes(b) if b is not None else None, fmt, o, enc)
    return bytes(out)[:160 if enc == ENC_LIMBS else 32], ok


def oracle_op(orc, o, P, Q=None):
    return {ADD: lambda: orc.add(P, Q), SUB: lambda: orc.sub(P, Q), NEG: lambda: orc.sub(orc.identity(), P),
            DOUBLE: lambda: orc.double(P), COFACTOR: lambda: orc.mul_by_pow_2(P, 3)}[o]()


def edwards_points(orc, torsion, rnd, k):
    B = orc.basepoint()
    pts = [orc.identity()] + [orc.p3_from_limbs(t["limbs"]) for t in torsion]
    pts += [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(k)]
    pts += [orc.add(orc.scalarmul(b32(rnd.randrange(L)), B), orc.p3_from_limbs(t["limbs"])) for t in torsion[:4]]
    return pts


def test_edwards_ops_against_the_oracle(host, orc, torsion):
    rnd = random.Random(31)
    pts = edwards_points(orc, torsion, rnd, 8)
    for i, P in enumerate(pts):
        Q = pts[rnd.randrange(len(pts))]
        for o in (ADD, SUB, NEG, DOUBLE, COFACTOR):
            want = oracle_op(orc, o, P, Q)
            got, ok = op(host, o, orc.compress(P), orc.compress(Q))
            assert (got, ok) == (orc.compress(want), 1), (i, o)
            got, ok = op(host, o, limbs_bytes(orc.p3_limbs(P)), limbs_bytes(orc.p3_limbs(Q)), EXTENDED, ENC_LIMBS)
            assert ok == 1 and orc.compress(orc.p3_from_limbs([int.from_bytes(got[8 * k:8 * k + 8], "little") for k in range(20)])) == \
                orc.compress(want), (i, o)


def test_p_plus_minus_p_and_add_against_double(host, orc, torsion):
    rnd = random.Random(32)
    for P in edwards_points(orc, torsion, rnd, 6):
        e = orc.compress(P)
        neg, _ = op(host, NEG, e)
        assert op(host, ADD, e, neg) == (b32(1), 1)
        assert op(host, SUB, e, e) == (b32(1), 1)
        assert op(host, ADD, e, e) == op(host, DOUBLE, e)
        assert host.h_eq(e, neg, COMPRESSED, 0) & 1 == (orc.compress(P) == orc.compress(orc.sub(orc.identity(), P)))


def test_small_order_points_and_identity(host, orc, torsion):
    for t in torsion:
        e = bytes.fromhex(t["compressed"])
        P = orc.p3_from_limbs(t["limbs"])
        assert op(host, COFACTOR, e) == (b32(1), 1)
        assert host.h_eq(e, None, COMPRESSED, 0) == (2 | int(orc.is_identity(P)))
        # every small-order point is in the Ristretto identity's coset exactly when it is 4-torsion
        four = orc.is_identity(orc.mul_by_pow_2(P, 2))
        assert host.h_eq(limbs_bytes(t["limbs"]), None, EXTENDED, 1) == (2 | int(four))


def test_non_canonical_edwards_encodings(host, orc):
    """y in [p, 2^255) decodes to the point of y - p, as the reference's decompress; equality is of points, not bytes."""
    hits = 0
    for y in range(19):
        for sign in (0, 1):
            enc = bytearray(b32(PRIME + y))
            enc[31] |= sign << 7
            canon = bytearray(b32(y))
            canon[31] |= sign << 7
            P = orc.decompress(bytes(enc))
            if P is None:
                assert op(host, DOUBLE, bytes(enc)) == (b32(1), 0)
                continue
            hits += 1
            assert host.h_eq(bytes(enc), bytes(canon), COMPRESSED, 0) == 3
            assert op(host, ADD, bytes(enc), bytes(canon)) == (orc.compress(orc.add(P, P)), 1)
            assert op(host, NEG, bytes(enc)) == (orc.compress(orc.sub(orc.identity(), P)), 1)
    assert hits >= 2


def test_undecodable_inputs(host, orc):
    good = orc.compress(orc.basepoint())
    assert op(host, ADD, b32(2), good) == (b32(1), 0)
    assert op(host, SUB, good, b32(2)) == (b32(1), 0)
    assert op(host, ADD, bytes(31) + b"\x80", good, RISTRETTO, ENC_RISTRETTO) == (bytes(32), 0)
    assert host.h_eq(b32(2), good, COMPRESSED, 0) == 0


def test_ristretto_ops_and_coset_equality(host, orc, torsion):
    rnd = random.Random(33)
    B = orc.basepoint()
    four = [orc.p3_from_limbs(t["limbs"]) for t in torsion]
    four = [T for T in four if orc.is_identity(orc.mul_by_pow_2(T, 2))]
    assert len(four) == 4
    for _ in range(8):
        P, Q = (orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(2))
        ep, eq_ = orc.ristretto_compress(P), orc.ristretto_compress(Q)
        for o in (ADD, SUB, NEG, DOUBLE):
            want = orc.ristretto_compress(oracle_op(orc, o, orc.ristretto_decompress(ep), orc.ristretto_decompress(eq_)))
            assert op(host, o, ep, eq_, RISTRETTO, ENC_RISTRETTO) == (want, 1)
        for T in four:
            PT = limbs_bytes(orc.p3_limbs(orc.add(P, T)))
            lp = limbs_bytes(orc.p3_limbs(P))
            assert host.h_eq(PT, lp, EXTENDED, 1) == 3                       # one Ristretto point
            assert host.h_eq(PT, lp, EXTENDED, 0) == (3 if orc.is_identity(T) else 2)   # distinct Edwards points
            assert op(host, ADD, PT, limbs_bytes(orc.p3_limbs(Q)), EXTENDED, ENC_RISTRETTO) == \
                (orc.ristretto_compress(orc.add(P, Q)), 1)


@pytest.mark.parametrize("threads", [1, 32, 128])
def test_sum(host, orc, torsion, threads):
    rnd = random.Random(34 + threads)
    pts = edwards_points(orc, torsion, rnd, 40)
    rnd.shuffle(pts)
    for n in (0, 1, 2, 31, 33, len(pts)):
        want = orc.identity()
        for P in pts[:n]:
            want = orc.add(want, P)
        out = (C.c_uint8 * 160)()
        enc = b"".join(orc.compress(P) for P in pts[:n]) or b"\0"
        assert host.h_sum(out, enc, n, COMPRESSED, threads, ENC_EDWARDS) == 1
        assert bytes(out)[:32] == orc.compress(want)
        ext = b"".join(limbs_bytes(orc.p3_limbs(P)) for P in pts[:n]) or b"\0"
        assert host.h_sum(out, ext, n, EXTENDED, threads, ENC_RISTRETTO) == 1
        assert bytes(out)[:32] == orc.ristretto_compress(want)
    bad = b"".join(orc.compress(P) for P in pts[:5]) + b32(2)
    out = (C.c_uint8 * 160)()
    assert host.h_sum(out, bad, 6, COMPRESSED, threads, ENC_EDWARDS) == 0 and bytes(out)[:32] == b32(1)


# ---- the chunk plan ----------------------------------------------------------------------------------------------------
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


def plan(host, sizes, chunk=CHUNK):
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    m = len(sizes)
    n_max = sum((s + chunk - 1) // chunk for s in sizes) + 1
    start, base, info = (C.c_uint32 * n_max)(), (C.c_uint32 * (m + 1))(), (C.c_uint32 * 3)()
    host.h_plan((C.c_uint64 * (m + 1))(*offs), m, chunk, start, base, info)
    return offs, list(start)[:info[0] + 1], list(base), info[1], info[2]


SHAPES = {
    "empty": [0], "one": [1], "empties_around": [0, 0, 5, 0, 0], "chunk_minus_1": [CHUNK - 1], "chunk": [CHUNK],
    "chunk_plus_1": [CHUNK + 1], "mixed": [0, 1, 2, 31, 32, 33, CHUNK - 1, CHUNK, CHUNK + 1, 0, 3 * CHUNK + 7],
    "straddle_pieces": [PIECE - 5, 1030, 7, PIECE + 3, 2 * PIECE - 1, 0, 1],
    "one_segment_of_many_pieces": [5 * PIECE + 3], "many_small": [16] * 5000, "many_ones": [1] * (PIECE + 17),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_chunk_plan_against_model(host, shape):
    sizes = SHAPES[shape]
    offs, start, base, max_len, max_per_seg = plan(host, sizes)
    assert (start, base, max_len, max_per_seg) == model_plan(offs, CHUNK)
    # every chunk lies inside one segment and the chunks of a segment tile it
    for j, (lo, hi) in enumerate(zip(offs[:-1], offs[1:])):
        cs = range(base[j], base[j + 1])
        assert all(lo <= start[c] < start[c + 1] <= hi and start[c + 1] - start[c] <= CHUNK for c in cs)
        assert (start[base[j]] if cs else lo) == lo and (start[base[j + 1]] if cs else hi) == hi
    # the pieces are runs of whole chunks of at most PIECE points, covering every chunk once
    nch = len(start) - 1
    cuts = (C.c_uint32 * (nch + 2))()
    k = host.h_pieces((C.c_uint32 * len(start))(*start), nch, PIECE, cuts)
    cuts = list(cuts)[:k]
    assert cuts == model_pieces(start, PIECE)
    assert cuts[0] == 0 and cuts[-1] == nch
    assert all(start[b] - start[a] <= PIECE and b > a for a, b in zip(cuts[:-1], cuts[1:]))
    # the next levels reduce every segment to at most one partial sum
    levels, b = 1, base
    while max_per_seg > 1:
        _, start2, b, _, max_per_seg = plan(host, [y - x for x, y in zip(b[:-1], b[1:])])
        levels += 1
    assert levels <= 3


# ---- SASS of the kernels -----------------------------------------------------------------------------------------------
# kernel -> (mangled name prefix, instantiations, bytes of stack frame as DESIGN.md section 9 records them: CUDA 12.9, sm_90a)
KERNELS = {"k_point_op": ("10k_point_opILi", 5, 0), "k_point_eq": ("10k_point_eqILi", 3, 0),
           "k_sum_decode": ("12k_sum_decodeILi", 3, 0), "k_sum_chunks": ("12k_sum_chunks", 1, 0),
           "k_sum_finish": ("12k_sum_finishILi", 2, 0)}


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
