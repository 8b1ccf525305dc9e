"""CPU tests (no GPU): an operator that halves its work after an OOM or at the 2^31-1 row limit does so through
`split_and_retry` (csrc/exec.cu), which also counts the split.  A split written out by hand would bring its own rules for
when to stop halving, so the sources may not contain one."""
import os

from tests.test_launch_sites import CSRC, _code, _without_function


def test_only_split_and_retry_counts_a_split():
    src = {}
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, name)) as fh:
                src[name] = _code(fh.read())
    assert src["exec.cu"].count("note_split(") == 1
    src["exec.cu"] = _without_function(src["exec.cu"], "static auto split_and_retry(")
    src["core.cu"] = _without_function(src["core.cu"], "void note_split()")
    src["common.cuh"] = src["common.cuh"].replace("void note_split();", "")
    for name, text in src.items():
        assert "note_split(" not in text, "%s counts a split by hand; use split_and_retry" % name
