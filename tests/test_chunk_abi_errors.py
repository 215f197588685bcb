"""The chunk entry points reject every argument the way the commit before their shared argument check did: the same
return code and error string, condition by condition and in the same order (``tests/golden/chunk_abi_errors.json``,
written by ``tests/golden/make_chunk_abi_errors.py``).  No call reaches the GPU."""
import importlib.util
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _make_errors():
    spec = importlib.util.spec_from_file_location("make_chunk_abi_errors",
                                                  os.path.join(GOLDEN, "make_chunk_abi_errors.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ME = _make_errors()
with open(os.path.join(GOLDEN, "chunk_abi_errors.json")) as _f:
    PARENT = json.load(_f)


@pytest.fixture(scope="module")
def nat():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


@pytest.mark.parametrize("entry", ME.ENTRIES)
def test_chunk_entry_point_rejects_as_parent(nat, entry):
    L, params = nat.lib(), ME.parameters()
    assert sorted(PARENT[entry]) == sorted(ME.key(c) for c in ME.CASES)
    got = {ME.key(c): ME.call(nat, L, params, entry, c) for c in ME.CASES}
    bad = {k: (got[k], v) for k, v in PARENT[entry].items() if got[k] != v}
    assert not bad, bad
