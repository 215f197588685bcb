"""ptxas report of the packed-document tile kernels (fwd_doc_sm90.cu, bwd_doc_sm90.cu): all 8 instantiations are
compiled, none serializes its wgmma pipeline (C7510 / "Performance Loss") and none spills."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "burst-attention_b200", "build")


@pytest.fixture(scope="module", autouse=True)
def built():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH) or not os.path.exists(os.path.join(BUILD, "bwd_doc_sm90.ptxas.log")):
        import __graft_entry__ as g
        g.build()


@pytest.mark.parametrize("tu,kern", [("fwd_doc_sm90", "fwd_doc_kernel"), ("bwd_doc_sm90", "bwd_doc_kernel")])
def test_doc_kernels_neither_serialize_nor_spill(tu, kern):
    log = open(os.path.join(BUILD, f"{tu}.ptxas.log")).read()
    assert "C7510" not in log and "Performance Loss" not in log, tu
    funcs = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len([f for f in funcs if kern in f]) == 4, funcs
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(a == "0" and b == "0" for a, b in spills), (tu, spills)
