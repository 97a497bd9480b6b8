"""Every kernel launch of the library goes through `lb::launch` (lasso_b200/csrc/common.cuh), which checks the launch
and counts it for `lasso_launch_count`.  A launch written with <<<...>>> anywhere else would go unchecked and
uncounted, and a hand-kept tally next to a launcher drifts from what the launcher does."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lasso_b200", "csrc")
HELPER = "common.cuh"


def _sources():
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".hpp", ".h", ".inc")):
            text = open(os.path.join(CSRC, name)).read()
            # comments may mention launches; only code counts
            text = re.sub(r"/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group()), text, flags=re.S)
            out[name] = re.sub(r"//[^\n]*", "", text)
    return out


def _helper_span(text):
    """(start, end) of the body of `launch` in common.cuh; empty without one"""
    m = re.search(r"\bvoid launch\(", text)
    if not m:
        return 0, 0
    start = text.index("{", m.end())
    depth = 0
    for i in range(start, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return start, i
    raise AssertionError("unbalanced braces in the launch helper")


def _line(text, pos):
    return text.count("\n", 0, pos) + 1


def test_every_launch_goes_through_the_helper():
    srcs = _sources()
    lo, hi = _helper_span(srcs[HELPER])
    bad = []
    for name, text in srcs.items():
        for m in re.finditer(r"<<<", text):
            if name == HELPER and lo < m.start() < hi:
                continue
            bad.append("%s:%d" % (name, _line(text, m.start())))
    assert not bad, "kernel launches outside lb::launch: " + ", ".join(bad)
    assert srcs[HELPER][lo:hi].count("<<<") == 1, "lb::launch is missing from common.cuh"


def test_only_the_helper_writes_the_launch_counter():
    srcs = _sources()
    lo, hi = _helper_span(srcs[HELPER])
    bad = []
    for name, text in srcs.items():
        for m in re.finditer(r"\bg_launches\b", text):
            rest = text[m.end():m.end() + 16]
            if name == HELPER and (lo < m.start() < hi or rest.startswith("{0}")):
                continue  # the helper's increment, and the definition
            if rest.startswith(".load()"):
                continue
            bad.append("%s:%d" % (name, _line(text, m.start())))
    assert not bad, "the launch counter is touched outside lb::launch: " + ", ".join(bad)
