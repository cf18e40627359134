"""CPU checks of the resident basepoint tables' kernels in the built library (sm_90a): no indirect branch (BRX/JMX), no
local memory, and stack frames no larger than DESIGN.md section 9 records; and the one comb-table builder left in the
library."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")

# kernel -> (mangled name prefix, instantiations, bytes of stack frame as DESIGN.md section 9 records them: CUDA 12.9,
# sm_90a).  The 32 bytes of k_bpt_mul<COMPRESSED> are register spills, not an indexed array.
KERNELS = {"k_comb_pow16": ("12k_comb_pow16ILi", 3, 0), "k_comb_rows": ("11k_comb_rowsP", 1, 0),
           "k_bpt_mul": ("9k_bpt_mulILi", 2, 32), "k_bpt_check_indices": ("19k_bpt_check_indicesP", 1, 0),
           "k_bpt_basepoints": ("16k_bpt_basepointsILi", 2, 0), "k_bpt_count": ("11k_bpt_countP", 1, 0),
           "k_bpt_offsets": ("13k_bpt_offsetsP", 1, 0), "k_bpt_order": ("11k_bpt_orderP", 1, 0)}


def _need_lib():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")


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


@pytest.fixture(scope="module")
def sass():
    _need_lib()
    return subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def usage():
    _need_lib()
    return subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines()


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_kernel_sass_has_no_indirect_branch(sass, kernel):
    name, count, _ = KERNELS[kernel]
    blocks = _function_sections(sass, name)
    assert len(blocks) == count, kernel
    for block in blocks:
        assert not re.search(r"\b(BRX|JMX)\b", block)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_kernel_resource_usage(usage, kernel):
    name, count, stack_max = KERNELS[kernel]
    idx = [i for i, l in enumerate(usage) if re.search(r"Function\s+\S*" + name, l)]
    assert len(idx) == count, kernel
    for i in idx:
        line = usage[i + 1]
        stack, local = re.search(r"\bSTACK:(\d+)\b", line), re.search(r"\bLOCAL:(\d+)\b", line)
        assert stack and local, line
        assert int(local.group(1)) == 0, line
        assert int(stack.group(1)) <= stack_max, line


def test_one_comb_table_builder(usage):
    """mul_batch's one-point comb and the resident tables share k_comb_pow16 + k_comb_rows"""
    assert not any("k_varmul_comb_table" in l for l in usage)


def test_design_records_the_figures():
    text = open(os.path.join(ROOT, "DESIGN.md")).read()
    for kernel, (_, _, stack) in KERNELS.items():
        m = re.search(r"^" + kernel + r"\b.*$", text, re.M)
        assert m, kernel
        assert ("%d bytes stack frame" % stack) in m.group(0) or (stack == 0 and "no stack" in m.group(0)), m.group(0)
