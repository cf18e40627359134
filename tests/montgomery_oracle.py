"""ctypes binding of the MontgomeryPoint CPU oracle (tests/host/montgomery_oracle.c, compiled together with the oracle
library's C sources).  TEST INFRASTRUCTURE ONLY: the parity source of the GPU MontgomeryPoint batches (Scalar *
MontgomeryPoint, mul_bits_be over up to 512 bits, to_edwards) and of the constant-time fixed-base batch.

The shared object is built with the system C compiler next to its source, or in a temporary directory when the tree is
read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "montgomery_oracle.c")
ODIR = os.path.join(ROOT, "oracle")
ORACLE_SRCS = ["fe51.c", "sc52.c", "curve.c", "msm.c", "hash.c", "ristretto.c", "batch.c", "parallel.c"]
FMT_COMPRESSED, FMT_RISTRETTO, FMT_MONTGOMERY = 0, 2, 3
_lib = None


def _deps():
    return [SRC] + [os.path.join(ODIR, f) for f in ORACLE_SRCS + ["oracle.h", "constants.h"]]


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-I", ODIR, "-o", so, SRC]
                          + [os.path.join(ODIR, f) for f in ORACLE_SRCS] + ["-lpthread"])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "libmontgomery_oracle.so")
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in _deps()):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="montgomery_oracle_"), "libmontgomery_oracle.so")
    _compile(so)
    return so


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        lib.mo_mul_bits_be.argtypes = [vp, vp, vp, C.c_uint, C.c_uint]
        lib.mo_mul_bits_be.restype = None
        lib.mo_to_edwards.argtypes = [vp, vp, C.c_uint8]
        lib.mo_to_edwards.restype = C.c_int
        lib.mo_mul_base.argtypes = [vp, vp, C.c_int, C.c_int]
        lib.mo_mul_base.restype = None
        lib.mo_mul_bits_be_batch.argtypes = [vp, vp, C.c_uint, sz, C.c_uint, vp, sz, sz]
        lib.mo_mul_bits_be_batch.restype = None
        lib.mo_to_edwards_batch.argtypes = [vp, vp, vp, vp, sz]
        lib.mo_to_edwards_batch.restype = sz
        lib.mo_mul_base_batch.argtypes = [vp, vp, sz, C.c_int, C.c_int]
        lib.mo_mul_base_batch.restype = None
        _lib = MontgomeryOracle(lib)
    return _lib


def _in(b):
    b = bytes(b)
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b if b else b"\0")


class MontgomeryOracle:
    def __init__(self, lib):
        self.lib = lib

    def mul_bits_be(self, u, b, nbits):
        """u([b] P) for the integer b (little-endian bytes, up to 64) read over bits nbits-1..0."""
        o = (C.c_uint8 * 32)()
        self.lib.mo_mul_bits_be(o, _in(u), _in(b), len(b), nbits)
        return bytes(o)

    def mul(self, s, u):
        """Scalar * MontgomeryPoint (s: 32 bytes, bit 255 clear)."""
        return self.mul_bits_be(u, s, 255)

    def to_edwards(self, u, sign):
        """CompressedEdwardsY of to_edwards(u, sign), or None."""
        o = (C.c_uint8 * 32)()
        return bytes(o) if self.lib.mo_to_edwards(o, _in(u), sign & 0xff) else None

    def mul_base(self, s, fmt, clamp=False):
        o = (C.c_uint8 * 32)()
        self.lib.mo_mul_base(o, _in(s), fmt, 1 if clamp else 0)
        return bytes(o)

    def mul_bits_be_batch(self, ints, int_bytes, n_ints, nbits, us, n_points, n):
        """flat inputs (n_ints / n_points each 1 or n) -> flat n x 32 bytes"""
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.mo_mul_bits_be_batch(o, _in(ints), int_bytes, n_ints, nbits, _in(us), n_points, n)
        return bytes(o)[:32 * n]

    def to_edwards_batch(self, us, signs, n):
        """-> (flat n x 32 bytes with the identity's encoding at None, n ok bytes)"""
        o, ok = (C.c_uint8 * (32 * max(n, 1)))(), (C.c_uint8 * max(n, 1))()
        self.lib.mo_to_edwards_batch(o, ok, _in(us), _in(signs), n)
        return bytes(o)[:32 * n], bytes(ok)[:n]

    def mul_base_batch(self, scalars, n, fmt, clamp=False):
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.mo_mul_base_batch(o, _in(scalars), n, fmt, 1 if clamp else 0)
        return bytes(o)[:32 * n]
