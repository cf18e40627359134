"""CPU checks of the verifying-key sets' kernels in the built library (sm_90a): the two instantiations of the front kernel
k_key_set_front use the registers, stack frame and local memory DESIGN.md section 9 records, and the per-key comb
kernels the sets reuse unchanged keep their figures (CUDA 12.9)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")

# mangled name -> (registers, bytes of stack frame); local memory is 0 for all
FRONT = {"_Z15k_key_set_frontILi0EE": (113, 0), "_Z15k_key_set_frontILi1EE": (122, 0)}
REUSED = {"_Z18k_verify_each_comb": (168, 752), "_Z16k_each_key_pow16": (168, 32), "_Z15k_each_key_rows": (232, 0)}


@pytest.fixture(scope="module")
def usage():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    lines = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines()
    out = {}
    for i, l in enumerate(lines):
        m = re.search(r"Function\s+(\S+?):?$", l.strip())
        if m:
            f = lines[i + 1]
            out[m.group(1)] = tuple(int(re.search(r"\b%s:(\d+)\b" % k, f).group(1)) for k in ("REG", "STACK", "LOCAL"))
    return out


def _one(usage, prefix):
    hits = [v for name, v in usage.items() if name.startswith(prefix)]
    assert len(hits) == 1, (prefix, hits)
    return hits[0]


@pytest.mark.parametrize("prefix", sorted(FRONT) + sorted(REUSED))
def test_kernel_resources(usage, prefix):
    reg, stack = {**FRONT, **REUSED}[prefix]
    assert _one(usage, prefix) == (reg, stack, 0)


def test_design_records_the_front_figures():
    text = open(os.path.join(ROOT, "DESIGN.md")).read()
    m = re.search(r"^k_key_set_front <0>, <1>\s+(\d+) / (\d+) registers, no stack, no local memory$", text, re.M)
    assert m, "DESIGN.md section 9 lists k_key_set_front's resources"
    assert (int(m.group(1)), int(m.group(2))) == (FRONT["_Z15k_key_set_frontILi0EE"][0], FRONT["_Z15k_key_set_frontILi1EE"][0])
