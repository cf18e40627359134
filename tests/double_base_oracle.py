"""ctypes binding of the double-base CPU oracle (tests/host/double_base_oracle.c, compiled together with the oracle
library's C sources).  TEST INFRASTRUCTURE ONLY: the parity source of the GPU double-base batch and the CPU baseline of
tools/bench_double_base.py.

Items are in the formats of the C ABI: a 64-byte scalar pair a || b and a point that is CompressedEdwardsY
(FMT_COMPRESSED), 160 bytes of radix-2^51 limbs (FMT_EXTENDED) or CompressedRistretto (FMT_RISTRETTO).  The shared
object is built with the system C compiler next to its source, or in a temporary directory when the tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "double_base_oracle.c")
ODIR = os.path.join(ROOT, "oracle")
ORACLE_SRCS = ["fe51.c", "sc52.c", "curve.c", "msm.c", "hash.c", "ristretto.c", "batch.c", "parallel.c"]
FMT_COMPRESSED, FMT_EXTENDED, FMT_RISTRETTO = 0, 1, 2
_lib = None


def _deps():
    return [SRC] + [os.path.join(ODIR, f) for f in ORACLE_SRCS + ["oracle.h", "constants.h"]]


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-I", ODIR, "-o", so, SRC]
                          + [os.path.join(ODIR, f) for f in ORACLE_SRCS] + ["-lpthread"])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "libdouble_base_oracle.so")
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in _deps()):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="double_base_oracle_"), "libdouble_base_oracle.so")
    _compile(so)
    return so


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        lib.dbo_one.argtypes = [vp, vp, vp, C.c_int, C.c_int]
        lib.dbo_one.restype = C.c_int
        lib.dbo_batch.argtypes = [vp, vp, vp, vp, C.c_int, sz, C.c_int]
        lib.dbo_batch.restype = C.c_int
        _lib = DoubleBaseOracle(lib)
    return _lib


def _in(b):
    b = bytes(b)
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b if b else b"\0")


class DoubleBaseOracle:
    def __init__(self, lib):
        self.lib = lib

    def one(self, a, point, b, fmt=FMT_COMPRESSED, naf=True):
        """(encoding of a A + b B, 1 if A decodes); naf=False: the oracle library's Straus-based value"""
        o = (C.c_uint8 * 32)()
        ok = self.lib.dbo_one(o, _in(bytes(a) + bytes(b)), _in(point), fmt, 1 if naf else 0)
        return bytes(o), ok

    def batch(self, ab, points, n, fmt=FMT_COMPRESSED, threads=1):
        """-> (rc 0 | 1 if some point does not decode, n x 32 bytes, n ok bytes); ab and points flat"""
        o, ok = (C.c_uint8 * (32 * max(n, 1)))(), (C.c_uint8 * max(n, 1))()
        rc = self.lib.dbo_batch(o, ok, _in(ab), _in(points), fmt, n, threads)
        return rc, bytes(o)[:32 * n], bytes(ok)[:n]
