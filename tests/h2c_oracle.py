"""ctypes binding of the hash-to-group CPU oracle (tests/host/h2c_oracle.c, compiled together with the oracle library's
C sources).  TEST INFRASTRUCTURE ONLY: the parity source of the GPU hash-to-group paths and the CPU baseline of
tools/bench_hash_to_curve.py.

The shared object is built with the system C compiler next to its source, or in a temporary directory when the tree
is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "h2c_oracle.c")
ODIR = os.path.join(ROOT, "oracle")
ORACLE_SRCS = ["fe51.c", "sc52.c", "curve.c", "msm.c", "hash.c", "ristretto.c", "batch.c", "parallel.c"]
CONSTANTS = ["ONE_MINUS_D_SQ", "D_MINUS_ONE_SQ", "SQRT_AD_MINUS_ONE", "MINUS_ONE", "MONTGOMERY_A", "MONTGOMERY_A_NEG",
             "SQRTAM2", "ELL2_C2", "EDWARDS_D", "SQRT_M1"]
_lib = None


def _deps():
    return [SRC] + [os.path.join(ODIR, f) for f in ORACLE_SRCS + ["oracle.h", "constants.h"]]


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-I", ODIR, "-o", so, SRC]
                          + [os.path.join(ODIR, f) for f in ORACLE_SRCS] + ["-lpthread"])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "libh2c_oracle.so")
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in _deps()):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="h2c_oracle_"), "libh2c_oracle.so")
    _compile(so)
    return so


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        lib.h2c_oracle_constant.argtypes = [vp, C.c_int]
        lib.h2c_ristretto_elligator.argtypes = [vp, vp]
        lib.h2c_from_uniform_bytes.argtypes = [vp, vp]
        lib.h2c_hash_from_bytes.argtypes = [vp, vp, sz]
        lib.h2c_from_bytes_wide.argtypes = [vp, vp]
        lib.h2c_expand_msg_xmd.argtypes = [vp, vp, sz, vp, sz, sz]
        lib.h2c_hash_to_field.argtypes = [vp, vp, sz, vp, sz, C.c_int]
        lib.h2c_map_to_curve.argtypes = [vp, vp]
        lib.h2c_hash_to_curve.argtypes = [vp, vp, sz, vp, sz, C.c_int]
        lib.h2c_flat_batch.argtypes = [vp, vp, vp, sz, vp, sz, C.c_int]
        lib.h2c_from_uniform_batch.argtypes = [vp, vp, sz]
        for f in ("h2c_oracle_constant", "h2c_ristretto_elligator", "h2c_from_uniform_bytes", "h2c_hash_from_bytes",
                  "h2c_from_bytes_wide", "h2c_expand_msg_xmd", "h2c_hash_to_field", "h2c_map_to_curve", "h2c_hash_to_curve",
                  "h2c_flat_batch", "h2c_from_uniform_batch"):
            getattr(lib, f).restype = None
        _lib = H2cOracle(lib)
    return _lib


def _in(b):
    b = bytes(b)
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b if b else b"\0")


class H2cOracle:
    def __init__(self, lib):
        self.lib = lib

    def constant(self, name):
        o = (C.c_uint8 * 32)(); self.lib.h2c_oracle_constant(o, CONSTANTS.index(name)); return bytes(o)

    def ristretto_elligator(self, r0):
        o = (C.c_uint8 * 32)(); self.lib.h2c_ristretto_elligator(o, _in(r0)); return bytes(o)

    def from_uniform_bytes(self, b):
        o = (C.c_uint8 * 32)(); self.lib.h2c_from_uniform_bytes(o, _in(b)); return bytes(o)

    def hash_from_bytes(self, m):
        o = (C.c_uint8 * 32)(); self.lib.h2c_hash_from_bytes(o, _in(m), len(m)); return bytes(o)

    def from_bytes_wide(self, b):
        o = (C.c_uint8 * 32)(); self.lib.h2c_from_bytes_wide(o, _in(b)); return bytes(o)

    def expand_message_xmd(self, m, dst, n):
        o = (C.c_uint8 * n)(); self.lib.h2c_expand_msg_xmd(o, _in(m), len(m), _in(dst), len(dst), n); return bytes(o)

    def hash_to_field(self, m, dst, count):
        o = (C.c_uint8 * (32 * count))(); self.lib.h2c_hash_to_field(o, _in(m), len(m), _in(dst), len(dst), count)
        return [bytes(o)[32 * i:32 * i + 32] for i in range(count)]

    def map_to_curve(self, u):
        o = (C.c_uint8 * 32)(); self.lib.h2c_map_to_curve(o, _in(u)); return bytes(o)

    def hash_to_curve(self, m, dst):
        o = (C.c_uint8 * 32)(); self.lib.h2c_hash_to_curve(o, _in(m), len(m), _in(dst), len(dst), 2); return bytes(o)

    def encode_to_curve(self, m, dst):
        o = (C.c_uint8 * 32)(); self.lib.h2c_hash_to_curve(o, _in(m), len(m), _in(dst), len(dst), 1); return bytes(o)

    def flat_batch(self, kind, msgs, dst=b"x"):
        """kind 'hash_from_bytes' | 'encode_to_curve' | 'hash_to_curve' over a list of messages -> list of encodings."""
        n = len(msgs)
        offs = (C.c_uint64 * (n + 1))()
        acc = 0
        for i, m in enumerate(msgs):
            offs[i] = acc; acc += len(m)
        offs[n] = acc
        o = (C.c_uint8 * (32 * max(n, 1)))()
        k = {"hash_from_bytes": 0, "encode_to_curve": 1, "hash_to_curve": 2}[kind]
        self.lib.h2c_flat_batch(o, _in(b"".join(msgs)), offs, n, _in(dst), len(dst), k)
        return [bytes(o)[32 * i:32 * i + 32] for i in range(n)]

    def from_uniform_batch(self, items):
        n = len(items)
        o = (C.c_uint8 * (32 * max(n, 1)))()
        self.lib.h2c_from_uniform_batch(o, _in(b"".join(items)), n)
        return [bytes(o)[32 * i:32 * i + 32] for i in range(n)]
