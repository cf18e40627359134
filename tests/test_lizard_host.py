"""Host build of the device Lizard code (csrc/lizard.cuh) with every fe.cuh limb-bound and fe64.cuh operand-scale
assertion on, against every golden vector and the model; decode's n_found == 2 branch through a table of fake digests; the
facts behind decode's shortcut (only the eight non-negative candidates are hashed); and the SASS of the Lizard kernels in
the built library.  CPU only."""
import ctypes as C
import hashlib
import json
import os
import random
import subprocess

import pytest

import h2c_model as H
import lizard_model as L
from test_hash_to_curve_host import _function_sections

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
KERNELS = ["k_ristretto_map_to_curve", "k_lizard_encode", "k_lizard_decodeILi1E", "k_lizard_decodeILi2E",
           "k_map_to_curve_inverseILi1E", "k_map_to_curve_inverseILi2E"]
FMT = {"extended": 1, "ristretto": 2}


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host", "lizard_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "liblizardhost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("lizard.cuh", "elligator.cuh", "ge.cuh", "fe64.cuh", "fe.cuh", "constants.cuh")]
    if not os.access(os.path.dirname(so), os.W_OK):
        so = str(tmp_path_factory.mktemp("lizardhost") / "liblizardhost.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    vp = C.c_void_p
    for f, a in (("h_sha256_16", [vp, vp]), ("h_map_to_curve", [vp, vp]), ("h_lizard_encode", [vp, vp]),
                 ("h_lizard_decode", [vp, vp, C.c_int]), ("h_map_to_curve_inverse", [vp, vp, C.c_int]),
                 ("h_to_jacobi", [vp, vp, C.c_int]), ("h_e_inv_positive", [vp, vp, vp]), ("h_fake_digest", [vp, vp]),
                 ("h_fake_clear", [])):
        getattr(lib, f).argtypes = a
    lib.h_fake_clear()
    yield lib
    lib.h_fake_clear()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "lizard.json")) as f:
        return json.load(f)


def call(fn, n, *args):
    o = (C.c_uint8 * n)()
    r = fn(o, *args)
    return r, bytes(o)


def decode(host, pt, fmt):
    return call(host.h_lizard_decode, 16, pt, fmt)


def inverse(host, pt, fmt):
    mask, raw = call(host.h_map_to_curve_inverse, 512, pt, fmt)
    return mask, [raw[32 * j:32 * j + 32] for j in range(16)]


def test_sha256_and_tag(host):
    rnd = random.Random(1)
    for _ in range(64):
        d = rnd.randbytes(16)
        assert call(host.h_sha256_16, 32, d)[1] == hashlib.sha256(d).digest()


def test_golden_encode_and_map(host, golden):
    for k in golden["lizard_encode_kat"]:
        assert call(host.h_lizard_encode, 32, bytes.fromhex(k["data"]))[1].hex() == k["out"]
    for v in golden["map_to_curve"]:
        assert call(host.h_map_to_curve, 32, bytes.fromhex(v["in"]))[1].hex() == v["out"], v["label"]
    h2c = json.load(open(os.path.join(ROOT, "tests", "golden", "hash_to_curve.json")))
    for v in h2c["ristretto_elligator_sage"]:
        assert call(host.h_map_to_curve, 32, bytes.fromhex(v["r0"]))[1].hex() == v["out"]
    for h in h2c["d_zero_halves"]:
        assert call(host.h_map_to_curve, 32, bytes.fromhex(h))[1] == H.ristretto_elligator(bytes.fromhex(h))


def test_golden_points(host, golden):
    for v in golden["points"]:
        pt, fmt = bytes.fromhex(v["point"]), FMT[v["fmt"]]
        n_found, data = decode(host, pt, fmt)
        assert n_found == (-1 if v["status"] == 2 else v["n_found"]), v["label"]
        assert data.hex() == (v["decode"] or "00" * 16), v["label"]
        mask, cands = inverse(host, pt, fmt)
        if v["status"] == 2:
            assert mask == -1, v["label"]                # the kernel zeroes the slots and the mask
            continue
        assert mask == v["mask"], v["label"]
        assert [c.hex() for c in cands] == [x or "00" * 32 for x in v["inverse"]], v["label"]


def test_golden_e_inv_positive(host, golden):
    for v in golden["e_inv_positive"]:
        some, out = call(host.h_e_inv_positive, 32, bytes.fromhex(v["s"]), bytes.fromhex(v["t"]))
        assert bool(some) == (v["out"] is not None), v["label"]
        assert out.hex() == (v["out"] or "00" * 32), v["label"]


def test_random_points_against_model(host):
    rnd = random.Random(2)
    for k in range(120):
        if k % 3 == 0:
            P = L.lizard_encode_point(rnd.randbytes(16))
        else:
            P = L.ristretto_decode(H.from_uniform_bytes(rnd.randbytes(64)))
        Q = L.scale(L.coset4(P)[rnd.randrange(4)], rnd.randrange(1, L.p))
        pt = L.limbs_bytes(Q)
        _, jac = call(host.h_to_jacobi, 256, pt, 1)
        want = L.to_jacobi_quartic(Q)
        assert [jac[32 * i:32 * i + 32] for i in range(8)] == [L.fe_bytes(x) for st in want for x in st]
        mask, cands = inverse(host, pt, 1)
        inv = L.map_to_curve_inverse(Q)
        assert cands == [x or bytes(32) for x in inv]
        assert mask == sum(1 << j for j, x in enumerate(inv) if x is not None)
        data, n_found, _ = L.lizard_decode_detail(Q)
        got_n, got = decode(host, pt, 1)
        assert got_n == n_found and got == (data or bytes(16))


def test_decode_shortcut_facts():
    """Decode hashes only the eight non-negative candidates.  The negated ones cannot pass the tag check: a negated
    candidate is odd unless it is zero (the check clears bit 0), and zero would need the masked SHA-256 of 16 zero bytes
    to be zero."""
    assert L.tag(bytes(16)) != bytes(32)
    rnd = random.Random(3)
    for _ in range(200):
        P = L.scale(L.map_to_curve_point(rnd.randbytes(32)), rnd.randrange(1, L.p))
        xs = L.elligator_inverse(P)
        for x in xs[:8]:
            assert x is None or x % 2 == 0
        for x in xs[8:]:
            assert x is None or x == 0 or x % 2 == 1
    # the identity's candidates include zero, and decode still finds nothing
    assert 0 in L.elligator_inverse(L.IDENTITY) and L.lizard_decode(L.IDENTITY) is None


def _two_taggable_candidates(rnd):
    """A point with two distinct non-negative candidates that a fake digest can make pass (bit 254 clear)."""
    while True:
        P = L.scale(L.ristretto_decode(H.from_uniform_bytes(rnd.randbytes(64))), rnd.randrange(1, L.p))
        xs = [x for x in L.elligator_inverse(P)[:8] if x is not None and x != 0 and not (x >> 254) & 1]
        xs = sorted(set(xs))
        if len(xs) >= 2 and L.fe_bytes(xs[0])[8:24] != L.fe_bytes(xs[1])[8:24]:
            return P, L.fe_bytes(xs[0]), L.fe_bytes(xs[1])


def test_two_passing_candidates_give_none(host):
    """n_found == 2 -> None: no real input reaches it (about 2^-122), so fake digests make two candidates of one point
    pass; with only one of them faked, decode returns that one's payload."""
    rnd = random.Random(4)
    try:
        for _ in range(3):
            P, b1, b2 = _two_taggable_candidates(rnd)
            pt = L.limbs_bytes(P)
            host.h_fake_clear()
            host.h_fake_digest(b1[8:24], b1)                 # tag(b1[8:24]) == b1
            n_found, data = decode(host, pt, 1)
            assert n_found == 1 and data == b1[8:24]
            host.h_fake_digest(b2[8:24], b2)
            n_found, data = decode(host, pt, 1)
            assert n_found == 2 and data == bytes(16)
            host.h_fake_clear()
            n_found, data = decode(host, pt, 1)
            assert n_found == 0 and data == bytes(16)
    finally:
        host.h_fake_clear()


@pytest.mark.parametrize("kernel", KERNELS)
def test_kernel_sass_has_no_indirect_branch(kernel):
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-sass", "-fun", kernel, LIB], capture_output=True, text=True)
    text = r.stdout if r.returncode == 0 and kernel in r.stdout else \
        subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    blocks = _function_sections(text, kernel)
    assert len(blocks) == 1
    assert "DFMA" in blocks[0]                  # the FP64 exponentiations
    assert not __import__("re").search(r"\b(BRX|JMX)\b", blocks[0])
