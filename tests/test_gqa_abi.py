"""CPU-side checks of the grouped-query entry points of the C-ABI: both are exported and bound, and a K/V head
count that is not positive or does not divide the query head count is rejected with an error string naming H_kv
before anything touches the GPU."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def nat():
    import os
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


def test_gqa_symbols_exported_and_bound(nat):
    L = ctypes.CDLL(nat.LIB_PATH)
    for name in ("ba_fwd_chunk_gqa", "ba_bwd_chunk_gqa"):
        assert hasattr(L, name), name
        assert name in nat.exported_symbols()
    assert nat.lib().ba_version() >= 201


@pytest.mark.parametrize("H,H_kv", [(32, 5), (4, 8), (8, 0), (8, -2)])
def test_bad_kv_head_count_returns_error_string(nat, H, H_kv):
    L = nat.lib()
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    rc = L.ba_fwd_chunk_gqa(z4, z4, z4, zr, z4, zr, z4, 1, 128, 128, H, H_kv, 128, 1.0, 0, 0, 3, 1, None)
    assert rc != 0 and b"H_kv" in L.ba_last_error()
    rc = L.ba_bwd_chunk_gqa(z4, z4, z4, z4, zr, zr, zr, z4, z4, z4, 1, 128, 128, H, H_kv, 128, 1.0, 0, 0, 0, 1, None)
    assert rc != 0 and b"H_kv" in L.ba_last_error()


def test_valid_kv_head_count_reaches_the_next_check(nat):
    """H % H_kv == 0 passes the head check: the call then fails on the null operands, not on H_kv."""
    L = nat.lib()
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    rc = L.ba_fwd_chunk_gqa(z4, z4, z4, zr, z4, zr, z4, 1, 128, 128, 32, 8, 128, 1.0, 0, 0, 3, 1, None)
    assert rc != 0 and b"null" in L.ba_last_error()
    rc = L.ba_bwd_chunk_gqa(z4, z4, z4, z4, zr, zr, zr, z4, z4, z4, 1, 128, 128, 32, 1, 128, 1.0, 0, 0, 0, 1, None)
    assert rc != 0 and b"null" in L.ba_last_error()
