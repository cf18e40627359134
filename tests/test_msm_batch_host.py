"""Host build of the device code of the batched MSMs (csrc/msm_batch.cuh) with the fe64 operand-scale assertions on:
the chunk loop of both modes against the C oracle, the cut of ragged MSM sizes into chunks against a Python model, and
the SASS / resource usage of the new kernels in the built library.  CPU only."""
import ctypes as C
import os
import random
import re
import subprocess

import pytest

import msm_digit_cases
import oracle_lib
import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
L = pyref.L
CHUNK_LENGTHS = [1, 2, 7, 8, 9, 16]


@pytest.fixture(scope="module")
def host():
    src = os.path.join(ROOT, "tests", "host", "msm_batch_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libmsmbatchhost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("msm_batch.cuh", "straus_vt.cuh", "warp4_f64.cuh", "ge64.cuh", "ge.cuh", "fe64.cuh",
                                                    "fe.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_mb_chunk.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    lib.h_mb_tasks.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.h_mb_tasks.restype = C.c_uint32
    lib.h_mb_radix16.argtypes = [C.c_void_p, C.c_char_p]
    return lib


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


def b32(x):
    return x.to_bytes(32, "little")


def chunk(host, scalars, encs, ct):
    out = (C.c_uint8 * 32)()
    ok = host.h_mb_chunk(out, b"".join(scalars), b"".join(encs), len(scalars), 1 if ct else 0)
    return bytes(out), ok


def want(orc, scalars, pts, ct):
    return orc.compress(orc.msm_ct(scalars, pts) if ct else orc.msm("straus_vartime", scalars, pts))


def test_chunk_length_is_sixteen(host):
    assert host.h_mb_chunk_max() == 16 == max(CHUNK_LENGTHS)


@pytest.mark.parametrize("ct", [False, True])
@pytest.mark.parametrize("n", CHUNK_LENGTHS)
def test_chunk_matches_oracle(host, orc, n, ct):
    rnd = random.Random(100 + n)
    B = orc.basepoint()
    pts = [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(n)]
    scalars = [b32(rnd.randrange(L)) if i % 2 else b32(rnd.randrange(2**255)) for i in range(n)]
    assert chunk(host, scalars, [orc.compress(p) for p in pts], ct) == (want(orc, scalars, pts, ct), 1)


@pytest.mark.parametrize("ct", [False, True])
def test_boundary_scalars(host, orc, ct):
    """The digit-boundary scalars of the bucket MSM at widths 4 and 5 (the widths of the two recodings) and the edge
    values below 2^255, sixteen to a chunk."""
    rnd = random.Random(7)
    B = orc.basepoint()
    vals = [s for c in (4, 5) for s in msm_digit_cases.boundary_scalars(c) if s < 2**255]
    for lo in range(0, len(vals), 16):
        scalars = [b32(s) for s in vals[lo:lo + 16]]
        pts = [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in scalars]
        assert chunk(host, scalars, [orc.compress(p) for p in pts], ct)[0] == want(orc, scalars, pts, ct)


@pytest.mark.parametrize("ct", [False, True])
def test_repeated_point_cancellation_and_identity(host, orc, ct):
    rnd = random.Random(8)
    B = orc.basepoint()
    P = orc.scalarmul(b32(rnd.randrange(L)), B)
    enc, ident = orc.compress(P), orc.compress(orc.identity())
    s = rnd.randrange(L)
    # the same point with the same scalar twice: the second addition is a doubling
    assert chunk(host, [b32(s), b32(s)], [enc, enc], ct)[0] == orc.compress(orc.scalarmul(b32(2 * s % L), P))
    # s P + (l - s) P = identity
    assert chunk(host, [b32(s), b32(L - s)], [enc, enc], ct)[0] == ident
    assert chunk(host, [b32(s), b32(5)], [ident, ident], ct)[0] == ident
    assert chunk(host, [b32(0)] * 3, [enc] * 3, ct)[0] == ident


def test_undecodable_point_is_reported(host):
    assert chunk(host, [b32(3)], [b32(2)], False)[1] == 0            # y = 2 is not on the curve


def test_radix16_digits(host, orc):
    rnd = random.Random(9)
    for s in [0, 1, L - 1, L, 2**255 - 1, 2**252] + [rnd.randrange(2**255) for _ in range(50)]:
        d = (C.c_int8 * 64)()
        host.h_mb_radix16(d, b32(s))
        assert list(d) == orc.radix16(b32(s))


def model_tasks(sizes, chunk_len=16):
    base, tasks, first = [0], [], 0
    for j, n in enumerate(sizes):
        k = (n + chunk_len - 1) // chunk_len
        base.append(base[-1] + k)
        tasks += [(j, first + chunk_len * i, min(chunk_len, n - chunk_len * i)) for i in range(k)]
        first += n
    return base, tasks


@pytest.mark.parametrize("sizes", [[0], [1], [16], [17], [0, 0, 0], [0, 5, 0, 0, 16, 1, 0], [33, 0, 32, 31, 0],
                                   [1000, 0, 0, 1, 499], "random"])
def test_task_list(host, sizes):
    if sizes == "random":
        rnd = random.Random(10)
        sizes = [rnd.choice([0, 0, 1, 2, 15, 16, 17, rnd.randrange(600)]) for _ in range(300)]
    offs = [0]
    for n in sizes:
        offs.append(offs[-1] + n)
    base, tasks = model_tasks(sizes)
    cap = len(tasks) + 1
    c_offs = (C.c_uint64 * len(offs))(*offs)
    c_base = (C.c_uint32 * len(offs))()
    seg, first, ln = (C.c_uint32 * cap)(), (C.c_uint64 * cap)(), (C.c_uint32 * cap)()
    n = host.h_mb_tasks(c_offs, len(sizes), c_base, seg, first, ln, cap)
    assert n == len(tasks) and list(c_base) == base
    assert [(seg[c], first[c], ln[c]) for c in range(n)] == tasks


def test_batch_symbols_are_declared_and_exported():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    header = open(os.path.join(ROOT, "include", "dalek_b200.h")).read()
    lib = C.CDLL(LIB)
    for name in ("dalek_b200_msm_batch", "dalek_b200_msm_batch_dev"):
        assert re.search(r"\bint %s\(" % name, header), name
        assert hasattr(lib, name), name


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


# the kernels a constant-time call runs: the chunk loop, the per-term preparation of each format, the finish of each
CT_KERNELS = {"11k_mb_chunksILb1E": 1, "12k_mb_prepareILi0ELb1E": 1, "12k_mb_prepareILi1ELb1E": 1, "12k_mb_prepareILi2ELb1E": 1,
              "11k_mb_finishILi": 3}


def test_constant_time_kernels_have_no_indirect_branch():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    for k, count in CT_KERNELS.items():
        blocks = _function_sections(r.stdout, k)
        assert len(blocks) == count, k
        for sass in blocks:
            assert "DFMA" in sass                    # the FP64 field
            assert not re.search(r"\b(BRX|JMX)\b", sass)


def test_chunk_kernels_resource_usage():
    """The constant-time chunk kernel keeps its accumulator, its selected entry and its digits in registers: no stack
    and no local memory.  The variable-time one keeps sixteen digit words (64 bytes) on its stack."""
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    seen = {}
    for i, l in enumerate(lines):
        m = re.search(r"Function\s+\S*11k_mb_chunksILb([01])E", l)
        if m:
            print(l.strip(), lines[i + 1].strip())
            seen[m.group(1)] = lines[i + 1]
    assert set(seen) == {"0", "1"}
    assert re.search(r"STACK:0\b", seen["1"]) and re.search(r"LOCAL:0\b", seen["1"])
    assert re.search(r"STACK:64\b", seen["0"]) and re.search(r"LOCAL:0\b", seen["0"])
    for usage in seen.values():
        assert int(re.search(r"REG:(\d+)", usage).group(1)) <= 192


@pytest.mark.parametrize("ct", [False, True])
@pytest.mark.parametrize("pattern", ["even", "ones", "small_odd"] + ["pow2_%d" % k for k in (2, 5, 6, 64, 200, 250)])
def test_chunk_scalar_patterns_shared_by_every_term(host, orc, pattern, ct):
    """Every scalar of the chunk even, a multiple of 2^k, or odd with one digit: no term adds in the last digit
    positions (or none ever doubles).  The chunk's sum is added to the other chunks of its MSM, so its T must be
    XY / Z (h_mb_chunk returns -2 otherwise)."""
    import straus_patterns as sp
    rnd = random.Random("%s-%d" % (pattern, ct))
    B = orc.basepoint()
    for n in (5, 16):
        pts = [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(n)]
        scalars = [b32(v) for v in sp.pattern_scalars(pattern, rnd, n)]
        assert chunk(host, scalars, [orc.compress(p) for p in pts], ct) == (want(orc, scalars, pts, ct), 1), n
