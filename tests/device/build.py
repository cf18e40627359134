"""Builds the TEST-ONLY device libraries tests/device/lib<name>.so (sm_90a, in-tree next to their sources).  Each compiles
product headers into a tiny harness; the product library does not contain them."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# harness -> the product headers it includes (directly or through another header)
TARGETS = {
    "fe_device_check": ("fe.cuh", "fe64.cuh"),                                   # tests/test_gpu_field.py
    "warp_device_check": ("fe.cuh", "fe64.cuh", "constants.cuh", "ge.cuh", "ge64.cuh", "warp4.cuh", "warp4_f64.cuh",
                          "x25519.cuh"),                                          # tests/test_gpu_warp_formulas.py
}


def _build_one(name):
    src = os.path.join(HERE, name + ".cu")
    out = os.path.join(HERE, "lib%s.so" % name)
    deps = [src, __file__] + [os.path.join(CSRC, f) for f in TARGETS[name]]
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in deps):
        return out
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
                           "-Xcompiler", "-fPIC", "-shared", "-o", out, src, "-lcudart"])
    return out


def build(name="fe_device_check"):
    """Builds every harness that is out of date and returns the path of `name`."""
    paths = {t: _build_one(t) for t in TARGETS}
    return paths[name]


if __name__ == "__main__":
    for t in TARGETS:
        print(_build_one(t))
