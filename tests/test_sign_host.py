"""CPU checks of the Ed25519 signer and Ed25519ph: the golden model against RFC 8032 7.3 and the C oracle, the host build
of the branch-free scalar arithmetic of csrc/sc.cuh against Python integers, and the SASS / local memory of the sign
kernels in the built library."""
import ctypes as C
import hashlib
import json
import os
import random
import re
import subprocess

import pytest

import ed25519ph_oracle
import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")
L = 2**252 + 27742317777372353535851937790883648493
MU = 2**512 // L

import sys  # noqa: E402
sys.path.insert(0, GOLDEN)
import make_ed25519ph_golden as model  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "ed25519ph.json")) as f:
        return json.load(f)


def test_model_reproduces_rfc8032_7_3():
    seed = bytes.fromhex(model.RFC_SEED)
    assert model.public_key(seed).hex() == model.RFC_PK
    assert model.sign_prehashed(seed, hashlib.sha512(b"abc").digest()).hex() == model.RFC_SIG


def test_fixture_is_what_the_generator_writes(golden):
    assert model.make() == golden


def test_oracle_agrees_with_every_fixture_vector(golden):
    o = ed25519ph_oracle.load()
    orc = oracle_lib.load()
    labels = set()
    for v in golden["vectors"]:
        labels.add(v["label"].rsplit("_", 1)[0])
        ph, ctx, sig, pk = (bytes.fromhex(v[k]) for k in ("prehash", "context", "sig", "pk"))
        if v["seed"]:
            seed = bytes.fromhex(v["seed"])
            assert orc.public_key(seed) == pk
            if v["verify"] == 0:
                assert o.sign_prehashed(seed, ph, ctx) == (0, sig), v["label"]
        assert o.verify_prehashed(ph, sig, pk, ctx) == v["verify"], v["label"]
        assert o.verify_prehashed(ph, sig, pk, ctx, strict=True) == v["verify_strict"], v["label"]
    assert {"rfc8032", "context_0", "context_1", "context_6", "context_255", "repudiation_prehash"} <= labels
    assert o.sign_prehashed(bytes(32), bytes(64), bytes(256))[0] == 5          # PrehashedContextLength


# ---- sc.cuh on the host ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sc():
    src = os.path.join(ROOT, "tests", "host", "sc_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libschost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("sc.cuh", "constants.cuh", "fe.cuh")]
    if not os.access(os.path.dirname(so), os.W_OK):
        import tempfile
        so = os.path.join(tempfile.mkdtemp(prefix="schost_"), "libschost.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    for f in ("h_sc_reduce512", "h_sc_mul", "h_sc_add", "h_sc_neg"):
        getattr(lib, f).restype = None
    return lib


def _buf(vals, nbytes):
    return (C.c_uint8 * max(1, nbytes * len(vals))).from_buffer_copy(b"".join(v.to_bytes(nbytes, "little") for v in vals) or b"\0")


def _out(buf, n):
    raw = bytes(buf)
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(n)]


def reduce512(lib, xs):
    o = (C.c_uint8 * (32 * len(xs)))()
    lib.h_sc_reduce512(o, _buf(xs, 64), C.c_size_t(len(xs)))
    return _out(o, len(xs))


def barrett_subtractions(x):
    """How many conditional subtractions of l the Barrett reduction of x (HAC 14.42, b = 2^32, k = 8) needs."""
    q3 = ((x >> 224) * MU) >> 288
    return ((x - q3 * L) % 2**288) // L


def test_sc_reduce512_edges_and_random(sc):
    rnd = random.Random(1)
    edges = [0, 1, L - 1, L, L + 1, 2 * L, 3 * L - 1, 2**252, 2**255 - 1, 2**256 - 1, 2**511, 2**512 - 1]
    # values whose Barrett estimate is short by one multiple of l (about one input in nine).  Short by two, which the
    # second masked subtraction covers, cannot happen for this l: the estimate misses q by at most
    # frac(2^512 / l) + 2^-28 + a floor < 0.23 + 2^-28 + 1 < 2 (checked below), so the second subtraction never fires.
    from fractions import Fraction
    assert Fraction(2**512, L) - MU < Fraction(1, 4)
    by1 = []
    while len(by1) < 256:
        x = rnd.randrange(2**512)
        assert barrett_subtractions(x) < 2
        if barrett_subtractions(x) == 1:
            by1.append(x)
    top = [(2**512 // L - j) * L + L - 1 for j in range(64)]          # the largest quotients
    assert all(barrett_subtractions(x) < 2 for x in top)
    xs = edges + by1 + [x for x in top if x < 2**512] + [rnd.randrange(2**512) for _ in range(100000)]
    assert reduce512(sc, xs) == [x % L for x in xs]


def test_sc_mul_add_neg(sc):
    rnd = random.Random(2)
    n = 100000
    edge = [0, 1, L - 1, L - 2, 2**252, (L - 1) // 2, (L + 1) // 2]
    a = edge + [rnd.randrange(L) for _ in range(n)]
    b = list(reversed(edge)) + [rnd.randrange(L) for _ in range(n)]
    m = len(a)
    o = (C.c_uint8 * (32 * m))()
    sc.h_sc_add(o, _buf(a, 32), _buf(b, 32), C.c_size_t(m))
    assert _out(o, m) == [(x + y) % L for x, y in zip(a, b)]
    sc.h_sc_neg(o, _buf(a, 32), C.c_size_t(m))
    assert _out(o, m) == [(-x) % L for x in a]
    # sc_mul takes any 256-bit operands (the signer multiplies by the clamped, unreduced a < 2^255)
    wa = [2**256 - 1, 2**255 - 1, L, 2 * L] + [rnd.randrange(2**256) for _ in range(n)]
    wb = [2**256 - 1, L - 1, 2**256 - 1, 3] + [rnd.randrange(2**256) for _ in range(n)]
    m = len(wa)
    o = (C.c_uint8 * (32 * m))()
    sc.h_sc_mul(o, _buf(wa, 32), _buf(wb, 32), C.c_size_t(m))
    assert _out(o, m) == [(x * y) % L for x, y in zip(wa, wb)]


# ---- SASS of the sign kernels ------------------------------------------------------------------------------------------
SIGN_KERNELS = {"k_sign_keys": "11k_sign_keys", "k_sign<0>": "6k_signILi0E", "k_sign<1>": "6k_signILi1E"}
# bytes of per-thread stack frame per kernel (where ptxas puts the register spills), as DESIGN.md section 9 records
# them (CUDA 12.9, sm_90a).  The spill slots can hold secrets (r, k a, s) in device memory that no call clears, so a
# growing frame is a change to review, not noise.
SIGN_STACK_MAX = {"k_sign_keys": 16, "k_sign<0>": 16, "k_sign<1>": 32}


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


@pytest.mark.parametrize("kernel", sorted(SIGN_KERNELS))
def test_sign_kernel_sass(kernel):
    _need_lib()
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    blocks = _function_sections(r.stdout, SIGN_KERNELS[kernel])
    assert len(blocks) == 1
    sass = blocks[0]
    assert "DFMA" in sass                        # the comb on the FP64 field
    assert not re.search(r"\b(BRX|JMX)\b", sass)
    assert "k_sign" in sass and "mul_base" not in sass


@pytest.mark.parametrize("kernel", sorted(SIGN_KERNELS))
def test_sign_kernel_spills(kernel):
    _need_lib()
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    idx = [i for i, l in enumerate(lines) if re.search(r"Function\s+\S*" + re.escape(SIGN_KERNELS[kernel]), l)]
    assert len(idx) == 1
    usage = lines[idx[0] + 1]
    stack, local = re.search(r"\bSTACK:(\d+)\b", usage), re.search(r"\bLOCAL:(\d+)\b", usage)
    assert stack and local, usage
    assert int(local.group(1)) == 0, usage                 # no local arrays: every register string is indexed statically
    assert int(stack.group(1)) <= SIGN_STACK_MAX[kernel], usage
