"""ctypes binding of the Ed25519ph CPU oracle (tests/host/ed25519ph_oracle.c, compiled together with the oracle library's
C sources).  TEST INFRASTRUCTURE ONLY: the parity source of the GPU Ed25519ph paths.

The shared object is built with the system C compiler next to its source, or in a temporary directory when the tree
is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "ed25519ph_oracle.c")
ODIR = os.path.join(ROOT, "oracle")
ORACLE_SRCS = ["fe51.c", "sc52.c", "curve.c", "msm.c", "hash.c", "ristretto.c", "batch.c", "parallel.c"]
_lib = None


def _deps():
    return [SRC] + [os.path.join(ODIR, f) for f in ORACLE_SRCS + ["oracle.h", "constants.h"]]


def _compile(so):
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-I", ODIR, "-o", so, SRC]
                          + [os.path.join(ODIR, f) for f in ORACLE_SRCS] + ["-lpthread"])


def build():
    """Compile the oracle next to its source if it is missing or stale; returns the path of the shared object."""
    so = os.path.join(ROOT, "tests", "host", "libed25519ph_oracle.so")
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in _deps()):
        return so
    if os.access(os.path.dirname(so), os.W_OK):
        _compile(so)
        return so
    so = os.path.join(tempfile.mkdtemp(prefix="ed25519ph_oracle_"), "libed25519ph_oracle.so")
    _compile(so)
    return so


def _in(b):
    b = bytes(b)
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b if b else b"\0")


class PhOracle:
    def __init__(self, lib):
        self.lib = lib
        vp, sz = C.c_void_p, C.c_size_t
        lib.ed25519ph_sign.argtypes = [vp, vp, vp, sz, vp]
        lib.ed25519ph_verify.argtypes = [vp, vp, sz, vp, vp, C.c_int]

    def sign_prehashed(self, seed, prehash, context=b""):
        """(rc, signature): rc 5 is PrehashedContextLength."""
        o = (C.c_uint8 * 64)()
        rc = self.lib.ed25519ph_sign(o, _in(prehash), _in(context), len(context), _in(seed))
        return rc, bytes(o)

    def verify_prehashed(self, prehash, sig, pk, context=b"", strict=False):
        return self.lib.ed25519ph_verify(_in(prehash), _in(context), len(context), _in(sig), _in(pk), 1 if strict else 0)


def load():
    global _lib
    if _lib is None:
        _lib = PhOracle(C.CDLL(build()))
    return _lib
