"""The stream-contract registry (tests/stream_cases.py) covers every stream-taking entry point of the C ABI: one case per prototype
of include/wispb200.h whose last parameter is `wb_stream s`, and no case for a function the header does not declare."""
import os
import re

import stream_cases

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "wispb200.h")


def stream_entry_points():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    decls = re.findall(r"\b(wb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src)
    assert len(decls) > 50, "header parse"
    return sorted(name for name, params in decls if re.search(r"\bwb_stream\s+s\s*$", params.strip()))


def test_every_stream_entry_point_has_a_case():
    want = stream_entry_points()
    missing = sorted(set(want) - set(stream_cases.CASES))
    unknown = sorted(set(stream_cases.CASES) - set(want))
    assert not missing, f"stream-taking entry points without a case in tests/stream_cases.py: {missing}"
    assert not unknown, f"cases naming no stream-taking entry point of the header: {unknown}"

