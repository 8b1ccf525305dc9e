"""CPU tests (no GPU): every kernel launch of the library goes through `launch()` (csrc/common.cuh), which raises the
kernel's dynamic shared-memory limit when needed, checks the launch and counts it.  A launch written out by hand
would skip some of that, so the sources may not contain one."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark-rapids_b200", "csrc")


def _code(text):
    """source without comments"""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _without_function(text, head):
    """`text` with every function definition that starts at `head` (its body found by brace matching) removed"""
    while True:
        i = text.find(head)
        if i < 0:
            return text
        j = text.index("{", i)
        depth = 0
        for k in range(j, len(text)):
            depth += {"{": 1, "}": -1}.get(text[k], 0)
            if depth == 0:
                break
        text = text[:i] + text[k + 1:]


def _sources_outside_helper():
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh")):
            continue
        with open(os.path.join(CSRC, name)) as fh:
            text = _code(fh.read())
        if name == "common.cuh":
            text = _without_function(text, "inline void launch(")
            text = text.replace("void count_launch();", "")
        if name == "core.cu":
            for head in ("void reserve_dyn_smem(", "void launch_done(", "void count_launch()"):
                text = _without_function(text, head)
        out[name] = text
    return out


def test_sources_are_found():
    src = _sources_outside_helper()
    assert {"common.cuh", "core.cu", "agg.cu", "prim.cuh", "exchange.cu"} <= set(src)
    with open(os.path.join(CSRC, "common.cuh")) as fh:
        assert "<<<" in _code(fh.read())


def test_kernels_launch_only_through_the_helper():
    for name, text in _sources_outside_helper().items():
        assert "<<<" not in text, "%s launches a kernel by hand; use launch()" % name
        assert "cudaFuncSetAttribute" not in text, "%s sets a kernel attribute by hand; launch() raises the shared-memory limit" % name


def test_only_nccl_work_is_counted_outside_the_helper():
    for name, text in _sources_outside_helper().items():
        lines = [ln.strip() for ln in text.splitlines() if "count_launch(" in ln]
        if name == "exchange.cu":
            assert lines == ["#define NCCL_LAUNCH(x) do { NCCL_CHECK(x); count_launch(); } while (0)"]
        else:
            assert lines == [], "%s counts launches by hand: %s" % (name, lines)
