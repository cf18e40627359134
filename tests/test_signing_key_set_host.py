"""CPU checks of hazmat signing and the signing-key sets: the raw_sign model (tests/raw_sign_model.py) reproduces the
Ed25519 test vectors and RFC 8032 7.3 when the ExpandedSecretKey is SHA-512(seed), and the kernel k_esk_keys in the built
library (sm_90a) runs the comb with no local memory and the stack frame DESIGN.md section 9 records."""
import hashlib
import json
import os
import re
import subprocess
import sys

import pytest

import oracle_lib
from raw_sign_model import RawSignModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")

# mangled-name prefix -> bytes of stack frame, as DESIGN.md section 9 records them (CUDA 12.9, sm_90a)
NEW_KERNELS = {"_Z10k_esk_keys": 16}


@pytest.fixture(scope="module")
def model():
    return RawSignModel(oracle_lib.load())


def test_model_reproduces_the_test_vectors(model):
    with open(os.path.join(GOLDEN, "ed25519_testvectors.json")) as f:
        tv = json.load(f)["vectors"]
    for v in tv:
        esk = hashlib.sha512(bytes.fromhex(v["seed"])).digest()
        vk = model.verifying_key(esk)
        assert vk.hex() == v["pk"], v["line"]
        assert model.raw_sign(esk, bytes.fromhex(v["msg"]), vk).hex() == v["sig"], v["line"]


def test_model_reproduces_rfc8032_7_3(model):
    sys.path.insert(0, GOLDEN)
    import make_ed25519ph_golden as ph
    esk = hashlib.sha512(bytes.fromhex(ph.RFC_SEED)).digest()
    vk = model.verifying_key(esk)
    assert vk.hex() == ph.RFC_PK
    assert model.raw_sign_prehashed(esk, hashlib.sha512(b"abc").digest(), vk).hex() == ph.RFC_SIG


def _usage():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    lines = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines()
    out = {}
    for i, l in enumerate(lines):
        m = re.search(r"Function\s+(\S+?):?$", l.strip())
        if m:
            f = lines[i + 1]
            out[m.group(1)] = tuple(int(re.search(r"\b%s:(\d+)\b" % k, f).group(1)) for k in ("STACK", "LOCAL"))
    return out


@pytest.mark.parametrize("prefix", sorted(NEW_KERNELS))
def test_new_kernel_resources(prefix):
    hits = [v for name, v in _usage().items() if name.startswith(prefix)]
    assert len(hits) == 1, hits
    stack, local = hits[0]
    assert local == 0
    assert stack <= NEW_KERNELS[prefix]


@pytest.mark.parametrize("prefix", sorted(NEW_KERNELS))
def test_new_kernel_runs_the_comb(prefix):
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    blocks, cur = [], None
    for line in sass.splitlines():
        m = re.search(r"Function\s*:\s*(\S+)", line)
        if m:
            cur = [] if m.group(1).startswith(prefix) else None
            if cur is not None:
                blocks.append(cur)
        if cur is not None:
            cur.append(line)
    assert len(blocks) == 1
    text = "\n".join(blocks[0])
    assert "DFMA" in text                                   # the comb on the FP64 field
    assert not re.search(r"\b(BRX|JMX)\b", text)


def test_design_records_the_new_frames():
    text = open(os.path.join(ROOT, "DESIGN.md")).read()
    m = re.search(r"^k_esk_keys\s+(\d+) registers, (\d+) bytes of stack, no local memory$", text, re.M)
    assert m, "DESIGN.md section 9 lists k_esk_keys's resources"
    assert int(m.group(2)) == NEW_KERNELS["_Z10k_esk_keys"]
