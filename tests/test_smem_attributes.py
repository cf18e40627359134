"""Every dynamic shared-memory limit the engine raises with cudaFuncSetAttribute is a named constant that does not change
between calls.

The limit belongs to the kernel on the device, so every context on the GPU shares it.  A value computed per call (from n,
the window width or the sort's fine bits) set by one context lowers the limit under a concurrent call of another context
that needs more, and that call's launch fails.  A scan of the sources, no GPU needed."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
HEADER = os.path.join(ROOT, "include", "dalek_b200.h")
TYPE_WORDS = {"int", "size_t", "sizeof", "double", "uint32_t", "uint64_t", "unsigned", "char"}
H100_MAX_DYN_SMEM = 227 * 1024                      # opt-in dynamic shared memory per block on sm_90


def _sources():
    paths = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    return {p: open(p).read() for p in paths + [HEADER]}


def _macros(texts):
    """NAME -> body of every object-like #define (line continuations joined, trailing // comment dropped)."""
    out = {}
    for text in texts.values():
        for m in re.finditer(r"^[ \t]*#define[ \t]+([A-Za-z_]\w*)(?!\()[ \t]*((?:.*\\\n)*.*)$", text, re.M):
            body = m.group(2).replace("\\\n", " ")
            out[m.group(1)] = re.sub(r"//.*", "", body).strip()
    return out


def _call_args(text, start):
    """Top-level comma-separated arguments of the call whose '(' is at text[start]."""
    depth, args, cur = 0, [], []
    for ch in text[start:]:
        if ch == "(":
            depth += 1
            if depth == 1:
                continue
        elif ch == ")":
            depth -= 1
            if depth == 0:
                args.append("".join(cur).strip())
                return args
        elif ch == "," and depth == 1:
            args.append("".join(cur).strip())
            cur = []
            continue
        cur.append(ch)
    raise AssertionError("unbalanced call")


def _smem_sites(texts):
    sites = []
    for path, text in texts.items():
        for m in re.finditer(r"\bcudaFuncSetAttribute\s*\(", text):
            args = _call_args(text, m.end() - 1)
            if args[-2] == "cudaFuncAttributeMaxDynamicSharedMemorySize":      # a template kernel's name may hold commas
                line = text.count("\n", 0, m.start()) + 1
                sites.append(("%s:%d" % (os.path.relpath(path, ROOT), line), ", ".join(args[:-2]), args[-1]))
    return sites


def _constant_value(expr, macros, seen=()):
    """The value of a constant expression of macros, literals and sizeof of a type; AssertionError if any name in it is
    not such a constant (a local variable, a parameter, a function)."""
    def name(m):
        w = m.group(0)
        if w in TYPE_WORDS:
            return w
        if w not in macros or w in seen:
            raise AssertionError("%r is not a named constant" % w)
        return "(%d)" % _constant_value(macros[w], macros, seen + (w,))
    e = re.sub(r"sizeof\s*\(\s*double\s*\)", "8", expr)
    e = re.sub(r"\b(\d+)[uUlL]+\b", r"\1", e)
    e = re.sub(r"[A-Za-z_]\w*", name, e)
    e = re.sub(r"\(\s*(int|size_t|uint32_t|uint64_t|unsigned)\s*\)", "", e)        # casts
    assert re.fullmatch(r"[\d\s()+\-*/<>%]+", e), "not a constant expression: %r" % expr
    return eval(e.replace("/", "//"))


def test_every_dynamic_smem_limit_is_a_named_call_independent_constant():
    texts = _sources()
    macros = _macros(texts)
    sites = _smem_sites(texts)
    assert len(sites) >= 9, sites                     # sort x 2, sign x 3, x25519, varmul, double-base comb, verify_each
    bad = []
    for where, kernel, expr in sites:
        names = [w for w in re.findall(r"[A-Za-z_]\w*", expr) if w not in TYPE_WORDS]
        try:
            assert names, "a bare literal"
            v = _constant_value(expr, macros)
            assert 0 < v <= H100_MAX_DYN_SMEM, "%d B is outside (0, %d]" % (v, H100_MAX_DYN_SMEM)
        except AssertionError as exc:
            bad.append("%s %s: %s (%s)" % (where, kernel, expr, exc))
    assert not bad, "\n".join(bad)


def test_digit_sort_limits_cover_every_fine_bits_choice():
    """The two sort kernels' limits are their sizes at the largest coarse-bin count and fine bits the sort can pick:
    nc <= SORT_NC_MAX coarse bins per window and F <= SORT_FINE_MAX fine bits."""
    texts = _sources()
    macros = _macros(texts)
    v = lambda name: _constant_value(name, macros)
    assert v("SORT_PART_SMEM_MAX") == v("SORT_TILE") * 8 + (2 * v("SORT_NC_MAX") + 33) * 4 == 49284
    assert v("SORT_FINE_SMEM_MAX") == v("SORT_FINE_CAP") * 12 + ((1 << v("SORT_FINE_MAX")) + 33) * 4 == 114820
