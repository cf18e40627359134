"""Host build of the device hash-to-group code (csrc/elligator.cuh) with every fe.cuh limb-bound and fe64.cuh operand-
scale assertion on, against the golden vectors, the model and map-level inputs that no hash reaches; and the SASS of the
hash-to-group kernels in the built library.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

import h2c_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
KERNELS = ["k_ristretto_from_uniform", "k_ristretto_hash_bytes", "k_edwards_h2cILi1E", "k_edwards_h2cILi2E"]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host", "h2c_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libh2chost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("elligator.cuh", "ge.cuh", "fe64.cuh", "fe.cuh", "constants.cuh")]
    if not os.access(os.path.dirname(so), os.W_OK):
        so = str(tmp_path_factory.mktemp("h2chost") / "libh2chost.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    for f, a in (("h_ristretto_elligator", [vp, vp]), ("h_from_uniform_bytes", [vp, vp]), ("h_hash_from_bytes", [vp, vp, sz]),
                 ("h_xmd", [vp, vp, sz, vp, C.c_uint32, C.c_int]), ("h_hash_to_field", [vp, vp, sz, vp, C.c_uint32, C.c_int]),
                 ("h_from_bytes_wide", [vp, vp]), ("h_ell2_encode", [vp, vp]), ("h_map_to_curve", [vp, vp]),
                 ("h_hash_to_curve", [vp, vp, sz, vp, C.c_uint32, C.c_int])):
        getattr(lib, f).argtypes = a
    return lib


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "hash_to_curve.json")) as f:
        return json.load(f)


def out(n):
    return (C.c_uint8 * n)()


def _b(x):
    x = bytes(x)
    return x if x else b"\0"


def call(host, name, n, *args):
    o = out(n)
    getattr(host, name)(o, *args)
    return bytes(o)


def test_ristretto_maps(host, golden):
    for v in golden["ristretto_elligator_sage"]:
        assert call(host, "h_ristretto_elligator", 32, bytes.fromhex(v["r0"])).hex() == v["out"]
    for v in golden["one_way_map"] + golden["from_uniform_edges"]:
        assert call(host, "h_from_uniform_bytes", 32, bytes.fromhex(v["in"])).hex() == v["out"], v.get("label")
    for v in golden["hash_from_bytes_lengths"]:
        m = bytes.fromhex(v["msg"])
        assert call(host, "h_hash_from_bytes", 32, _b(m), len(m)).hex() == v["out"], v["label"]


def test_field_and_xmd(host, golden):
    ro, nu = bytes.fromhex(golden["dst_ro"]), bytes.fromhex(golden["dst_nu"])
    for v in golden["from_bytes_wide"]:
        assert call(host, "h_from_bytes_wide", 32, bytes.fromhex(v["in"])).hex() == v["out"]
    rnd = random.Random(1)
    for _ in range(200):
        b = rnd.randbytes(64)
        assert call(host, "h_from_bytes_wide", 32, b) == M.from_bytes_wide(b).to_bytes(32, "little")
    for key, dst, count in (("rfc9380_hash_to_field_1", nu, 1), ("rfc9380_hash_to_field_2", ro, 2)):
        for v in golden[key]:
            m = bytes.fromhex(v["msg"])
            got = call(host, "h_hash_to_field", 32 * count, _b(m), len(m), dst, len(dst), count)
            assert [got[32 * i:32 * i + 32].hex() for i in range(count)] == v["u"]
    for v in golden["xmd_boundaries"]:
        m, dst = bytes.fromhex(v["msg"]), bytes.fromhex(v["dst"])
        assert call(host, "h_xmd", 48, _b(m), len(m), dst, len(dst), 1).hex() == v["uniform_48"], v["label"]
        assert call(host, "h_xmd", 96, _b(m), len(m), dst, len(dst), 2).hex() == v["uniform_96"], v["label"]


def test_edwards_hash_and_encode(host, golden):
    ro, nu = bytes.fromhex(golden["dst_ro"]), bytes.fromhex(golden["dst_nu"])
    for key, dst, count in (("rfc9380_hash_to_curve", ro, 2), ("rfc9380_encode_to_curve", nu, 1)):
        for v in golden[key]:
            m = bytes.fromhex(v["msg"])
            assert call(host, "h_hash_to_curve", 32, _b(m), len(m), dst, len(dst), count).hex() == v["out"]
    for v in golden["xmd_boundaries"]:
        m, dst = bytes.fromhex(v["msg"]), bytes.fromhex(v["dst"])
        assert call(host, "h_hash_to_curve", 32, _b(m), len(m), dst, len(dst), 2).hex() == v["hash_to_curve"]
        assert call(host, "h_hash_to_curve", 32, _b(m), len(m), dst, len(dst), 1).hex() == v["encode_to_curve"]


def test_map_level_inputs(host, golden):
    """u = 0 reaches the tv1 == 0 exceptional case (the 2-torsion point (0, 0) of curve25519 maps to the identity)."""
    seen_exceptional = False
    for v in golden["map_to_curve"]:
        o = out(32)
        flag = host.h_map_to_curve(o, bytes.fromhex(v["u"]))
        assert bytes(o).hex() == v["out"], v["label"]
        assert bool(flag) == v["exceptional"], v["label"]
        seen_exceptional |= bool(flag)
    assert seen_exceptional
    enc = call(host, "h_ell2_encode", 96, bytes(32))
    assert enc[:32] == bytes(32) and enc[64:] == bytes(32)          # u = 0 -> (0, 0) on curve25519
    rnd = random.Random(2)
    for _ in range(300):
        u = rnd.randrange(M.p)
        o = out(32)
        host.h_map_to_curve(o, u.to_bytes(32, "little"))
        assert bytes(o) == M.map_to_curve_compressed(u)


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
    assert not re.search(r"\b(BRX|JMX)\b", blocks[0])
