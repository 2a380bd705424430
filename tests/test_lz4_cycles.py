"""The team encoder's cycle counters (dev_lz4.cuh, enum LZ4C_*) and scripts/lz4_cycles.py, which reads them by
column index, must agree on the layout."""
import importlib.util
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cycle_columns_match_the_device_enum():
    src = open(os.path.join(ROOT, "c-blosc_b200", "csrc", "dev_lz4.cuh")).read()
    body = re.search(r"enum \{\s*(LZ4C_TOTAL.*?)\};", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [t.strip() for t in body.split(",") if t.strip()]
    assert names[-1] == "LZ4C_N = 16"
    cols = [n[len("LZ4C_"):] for n in names[:-1]]
    spec = importlib.util.spec_from_file_location("lz4_cycles", os.path.join(ROOT, "scripts", "lz4_cycles.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.NCOL == 16 and len(cols) <= mod.NCOL
    for i, c in enumerate(cols):
        assert getattr(mod, c) == i, c
    assert re.search(r"#define LZ4C_MAXSTREAMS %d\b" % mod.MAXSTREAMS, src)
