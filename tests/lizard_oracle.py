"""ctypes binding of the Lizard CPU oracle (tests/host/lizard_oracle.c, compiled together with tests/host/h2c_oracle.c and
the oracle library's C sources).  TEST INFRASTRUCTURE ONLY: the parity source of the GPU Lizard paths and the CPU baseline
of tools/bench_lizard.py.

Points are CompressedRistretto (FMT_RISTRETTO) or 160 bytes of radix-2^51 limbs of one representative (FMT_EXTENDED),
the formats of the C ABI.  The shared object is built with the system C compiler next to its source, or in a temporary
directory when the tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "lizard_oracle.c")
H2C_SRC = os.path.join(ROOT, "tests", "host", "h2c_oracle.c")
ODIR = os.path.join(ROOT, "oracle")
ORACLE_SRCS = ["fe51.c", "sc52.c", "curve.c", "msm.c", "hash.c", "ristretto.c", "batch.c", "parallel.c"]
CONSTANTS = ["SQRT_ID", "DP1_OVER_DM1", "MDOUBLE_INVSQRT_A_MINUS_D", "MIDOUBLE_INVSQRT_A_MINUS_D", "MINVSQRT_ONE_PLUS_D",
             "SQRT_M1", "MINUS_ONE"]
FMT_EXTENDED, FMT_RISTRETTO = 1, 2          # DALEK_POINTS_EXTENDED / DALEK_POINTS_RISTRETTO
_lib = None


def _deps():
    return [SRC, H2C_SRC] + [os.path.join(ODIR, f) for f in ORACLE_SRCS + ["oracle.h", "constants.h"]]


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-I", ODIR, "-o", so, SRC, H2C_SRC]
                          + [os.path.join(ODIR, f) for f in ORACLE_SRCS] + ["-lpthread"])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "liblizard_oracle.so")
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in _deps()):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="lizard_oracle_"), "liblizard_oracle.so")
    _compile(so)
    return so


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        lib.lz_constant.argtypes = [vp, C.c_int]
        lib.lz_sha256.argtypes = [vp, vp, sz]
        lib.lz_encode.argtypes = [vp, vp]
        lib.lz_decode.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        lib.lz_decode.restype = C.c_int
        lib.lz_map_to_curve_inverse.argtypes = [vp, vp, vp, C.c_int]
        lib.lz_map_to_curve_inverse.restype = C.c_int
        lib.lz_encode_batch.argtypes = [vp, vp, sz]
        lib.lz_map_to_curve_batch.argtypes = [vp, vp, sz]
        lib.lz_decode_batch.argtypes = [vp, vp, vp, C.c_int, sz]
        lib.lz_map_to_curve_inverse_batch.argtypes = [vp, vp, vp, C.c_int, sz]
        for f in ("lz_constant", "lz_sha256", "lz_encode", "lz_encode_batch", "lz_map_to_curve_batch", "lz_decode_batch",
                  "lz_map_to_curve_inverse_batch"):
            getattr(lib, f).restype = None
        _lib = LizardOracle(lib)
    return _lib


def _in(b):
    b = bytes(b)
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b if b else b"\0")


class LizardOracle:
    def __init__(self, lib):
        self.lib = lib

    def constant(self, name):
        o = (C.c_uint8 * 32)(); self.lib.lz_constant(o, CONSTANTS.index(name)); return bytes(o)

    def sha256(self, m):
        o = (C.c_uint8 * 32)(); self.lib.lz_sha256(o, _in(m), len(m)); return bytes(o)

    def lizard_encode(self, data):
        o = (C.c_uint8 * 32)(); self.lib.lz_encode(o, _in(data)); return bytes(o)

    def lizard_decode(self, pt, fmt=FMT_RISTRETTO):
        """(status 0 Some | 1 None | 2 undecodable, 16-byte payload (zero unless Some), n_found)"""
        o, nf = (C.c_uint8 * 16)(), C.c_int()
        st = self.lib.lz_decode(o, _in(pt), fmt, C.byref(nf))
        return st, bytes(o), nf.value

    def map_to_curve_inverse(self, pt, fmt=FMT_RISTRETTO):
        """(undecodable flag, 16 x 32 bytes (zero where None), mask)"""
        o, m = (C.c_uint8 * 512)(), C.c_uint16()
        bad = self.lib.lz_map_to_curve_inverse(o, C.byref(m), _in(pt), fmt)
        return bad, [bytes(o)[32 * j:32 * j + 32] for j in range(16)], m.value

    def lizard_encode_batch(self, items):
        n = len(items)
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.lz_encode_batch(o, _in(b"".join(items)), n)
        return [bytes(o)[32 * i:32 * i + 32] for i in range(n)]

    def map_to_curve_batch(self, items):
        n = len(items)
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.lz_map_to_curve_batch(o, _in(b"".join(items)), n)
        return [bytes(o)[32 * i:32 * i + 32] for i in range(n)]

    def lizard_decode_batch(self, pts, fmt=FMT_RISTRETTO):
        """-> (flat n x 16 payload bytes, n status bytes)"""
        n = len(pts)
        o, st = (C.c_uint8 * (16 * max(n, 1)))(), (C.c_uint8 * max(n, 1))()
        self.lib.lz_decode_batch(o, st, _in(b"".join(pts)), fmt, n)
        return bytes(o)[:16 * n], bytes(st)[:n]

    def map_to_curve_inverse_batch(self, pts, fmt=FMT_RISTRETTO):
        """-> (flat n x 512 candidate bytes, list of n masks)"""
        n = len(pts)
        o, m = (C.c_uint8 * (512 * max(n, 1)))(), (C.c_uint16 * max(n, 1))()
        self.lib.lz_map_to_curve_inverse_batch(o, m, _in(b"".join(pts)), fmt, n)
        return bytes(o)[:512 * n], list(m)[:n]
