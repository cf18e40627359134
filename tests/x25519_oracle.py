"""ctypes binding of the X25519 CPU oracle (tests/host/x25519_oracle.c).  TEST INFRASTRUCTURE ONLY: the parity
source of the GPU X25519 paths and the one-core CPU baseline of tools/bench_x25519.py.

The shared object is built with the system C compiler next to its source, or in a temporary directory when the
tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "x25519_oracle.c")
_lib = None


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-Wall", "-fPIC", "-shared", "-o", so, SRC])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "libx25519_oracle.so")
    if os.path.exists(so) and os.path.getmtime(so) >= os.path.getmtime(SRC):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="x25519_oracle_"), "libx25519_oracle.so")
    _compile(so)
    return so


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp = C.c_void_p
        lib.x25519_clamp_integer.argtypes = [vp, vp]
        lib.x25519_mul_bits_be.argtypes = [vp, vp, vp, C.c_uint]
        lib.x25519_scalarmult.argtypes = [vp, vp, vp]
        lib.x25519_scalarmult_batch.argtypes = [vp, vp, vp, C.c_size_t]
        lib.x25519_edwards_to_montgomery.argtypes = [vp, vp]
        for f in ("x25519_clamp_integer", "x25519_mul_bits_be", "x25519_scalarmult", "x25519_scalarmult_batch",
                  "x25519_edwards_to_montgomery"):
            getattr(lib, f).restype = None
        _lib = X25519Oracle(lib)
    return _lib


def _in(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(bytes(b) if b else b"\0")


class X25519Oracle:
    def __init__(self, lib):
        self.lib = lib

    def clamp(self, k):
        o = (C.c_uint8 * 32)(); self.lib.x25519_clamp_integer(o, _in(k)); return bytes(o)

    def mul_bits_be(self, u, scalar, nbits):
        o = (C.c_uint8 * 32)(); self.lib.x25519_mul_bits_be(o, _in(u), _in(scalar), nbits); return bytes(o)

    def x25519(self, k, u):
        o = (C.c_uint8 * 32)(); self.lib.x25519_scalarmult(o, _in(k), _in(u)); return bytes(o)

    def x25519_batch(self, ks, us):
        """ks, us: flat n x 32-byte buffers -> flat n x 32 bytes."""
        n = len(ks) // 32
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.x25519_scalarmult_batch(o, _in(ks), _in(us), n)
        return bytes(o)[:32 * n]

    def public_key(self, k):
        return self.x25519(k, bytes([9]) + bytes(31))

    def to_montgomery(self, limbs):
        o = (C.c_uint8 * 32)()
        self.lib.x25519_edwards_to_montgomery(o, (C.c_uint64 * 20)(*limbs))
        return bytes(o)
