"""Every device workspace of a context has one role (enum WsRole in engine.h), and each role's comment names the files
that may use it, the owner first, and the lifetime of its contents.  Two files that reach for the same workspace without
the role saying so could overwrite each other's data between calls or inside a nested call.  A scan of the sources, no
GPU needed."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
ENGINE_H = os.path.join(CSRC, "engine.h")
LIFETIMES = {"call", "cross-call", "context"}


def _sources():
    paths = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    return {os.path.basename(p): open(p).read() for p in paths}


def _roles():
    """role -> (allowed files, lifetime), from the comment above each enumerator of WsRole."""
    text = open(ENGINE_H).read()
    body = re.search(r"\benum WsRole\s*\{(.*?)\};", text, re.S).group(1)
    roles, comment = {}, []
    for line in body.split("\n"):
        line = line.strip()
        if line.startswith("// ----"):
            comment = []
        elif line.startswith("//"):
            comment.append(line[2:].strip())
        elif re.fullmatch(r"WS_\w+,?", line):
            name = line.rstrip(",")
            if name == "WS_COUNT":
                continue
            m = re.match(r"((?:[\w.]+\.(?:cu|cuh|h),?\s*)+)\[([\w-]+)\]", " ".join(comment))
            assert m, "%s: the comment does not start with its files and [lifetime]: %r" % (name, comment)
            files = re.findall(r"[\w.]+\.(?:cu|cuh|h)", m.group(1))
            roles[name] = (files, m.group(2))
            comment = []
        elif line:
            raise AssertionError("unexpected line in enum WsRole: %r" % line)
    return roles


def _uses(texts):
    """(file, line, role) of every ctx->ws[...] in the sources."""
    out = []
    for name, text in texts.items():
        for m in re.finditer(r"ctx->ws\[([^\]]*)\]", text):
            line = text.count("\n", 0, m.start()) + 1
            for role in re.findall(r"\bWS_\w+", m.group(1)):
                out.append((name, line, role))
    return out


def test_every_role_names_its_files_and_lifetime():
    roles = _roles()
    assert len(roles) >= 40, sorted(roles)
    texts = _sources()
    for name, (files, lifetime) in roles.items():
        assert lifetime in LIFETIMES, (name, lifetime)
        for f in files:
            assert f in texts, "%s names %s, which is not a source file" % (name, f)


def test_every_workspace_use_is_in_a_file_its_role_allows():
    roles = _roles()
    bad = []
    for f, line, role in _uses(_sources()):
        if role not in roles:
            bad.append("%s:%d: %s is not a role" % (f, line, role))
        elif f not in roles[role][0]:
            bad.append("%s:%d: %s is only for %s" % (f, line, role, ", ".join(roles[role][0])))
    assert not bad, "\n".join(bad)


def test_no_role_is_left_unused():
    used = {role for _, _, role in _uses(_sources())}
    assert not set(_roles()) - used, sorted(set(_roles()) - used)


def test_the_context_holds_no_device_workspace_outside_the_array():
    text = open(ENGINE_H).read()
    body = re.search(r"\bstruct dalek_b200_ctx\s*\{(.*?)\n\};", text, re.S).group(1)
    fields = [l.strip() for l in body.split("\n") if re.match(r"\s*DevBuf\b", l)]
    assert len(fields) == 1 and re.match(r"DevBuf ws\[WS_COUNT\];", fields[0]), fields


def test_status_words_are_named_slots():
    """WS_FLAGS carries words of different calls; an offset into it is one of the FLAG_* slots, never a bare number."""
    bad = []
    for name, text in _sources().items():
        for m in re.finditer(r"ctx->ws\[WS_FLAGS\]\.p\s*\)?\s*\+\s*(\w+)", text):
            if not m.group(1).startswith("FLAG_"):
                bad.append("%s:%d: %s" % (name, text.count("\n", 0, m.start()) + 1, m.group(0)))
        for m in re.finditer(r"\bflags\[(\w+)\]", text):
            if not m.group(1).startswith("FLAG_"):
                bad.append("%s:%d: %s" % (name, text.count("\n", 0, m.start()) + 1, m.group(0)))
    assert not bad, "\n".join(bad)
