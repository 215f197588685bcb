"""CPU-side checks of the C-ABI boundary: the shared library loads, exports every
symbol include/burst_attn_b200.h declares, its ctypes binding has the header's
signatures, and it rejects bad arguments with an error string instead of
crashing.  No compute call is made (no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "burst_attn_b200.h")
SELFTEST_HEADER = os.path.join(ROOT, "include", "burst_attn_b200_selftest.h")


def _declared():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"\b(ba_[a-z0-9_]+)\s*\(", src)))


def _prototypes(path):
    """{name: (return type, [parameter types])} of the functions a C header declares, types with their names
    dropped and whitespace normalised, e.g. "const void* const*"."""
    src = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(path).read(), flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    out = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w\s*]*?)\s*\b(ba_\w+)\s*\(([^)]*)\)\s*;", src):
        params = [] if params.strip() == "void" else [p.strip() for p in params.split(",")]
        types = [" ".join(re.sub(r"\*", " * ", re.sub(r"\s*\w+$", "", p)).split()).replace(" *", "*")
                 for p in params]
        out[name] = (" ".join(ret.split()), types)
    return out


def _ctype(nat, c_type, ret=False):
    """The ctypes type a C type maps to: structs by value, scalars, and pointers as c_void_p except
    int64_t* (POINTER(c_int64)), pointers to pointers (POINTER(c_void_p)) and a returned string."""
    base = " ".join(w for w in c_type.replace("*", " ").split() if w != "const")
    depth = c_type.count("*")
    if ret and c_type == "const char*":
        return ctypes.c_char_p
    if depth == 0:
        return {"int": ctypes.c_int, "float": ctypes.c_float, "int64_t": ctypes.c_int64,
                "ba_tensor4": nat.ba_tensor4, "ba_rowstat": nat.ba_rowstat}[base]
    if depth == 1:
        return ctypes.POINTER(ctypes.c_int64) if base == "int64_t" else ctypes.c_void_p
    assert depth == 2, c_type
    return ctypes.POINTER(ctypes.c_void_p)


@pytest.fixture(scope="module")
def nat():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


def test_header_and_binding_agree(nat):
    assert _declared() == sorted(nat.exported_symbols())


def test_library_exports_every_declared_symbol(nat):
    L = ctypes.CDLL(nat.LIB_PATH)
    for name in _declared():
        assert hasattr(L, name), name


def test_selftest_library_is_separate_from_the_product(nat):
    """Diagnostics (ba_selftest) live in their own header and library, not in the drop-in boundary."""
    hdr = open(os.path.join(ROOT, "include", "burst_attn_b200_selftest.h")).read()
    declared = sorted(set(re.findall(r"\b(ba_[a-z0-9_]+)\s*\(", hdr)))
    assert declared == sorted(nat._SELFTEST_EXPORTS)
    T = ctypes.CDLL(nat.SELFTEST_LIB_PATH)
    for name in declared:
        assert hasattr(T, name), name
    L = ctypes.CDLL(nat.LIB_PATH)
    for name in ("ba_selftest", "ba_selftest_last_error"):
        assert not hasattr(L, name), f"{name} must not be exported by the product library"


def test_binding_signatures_match_header(nat):
    """Every bound function's restype and argtypes are the ctypes form of its prototype in the header: ctypes
    itself checks neither, so a wrong or missing argument type would pass garbage to the library."""
    for header, L in ((HEADER, nat.lib()), (SELFTEST_HEADER, nat.selftest_lib())):
        protos = _prototypes(header)
        assert protos, header
        for name, (ret, params) in protos.items():
            fn = getattr(L, name)
            assert fn.restype is _ctype(nat, ret, ret=True), (name, ret, fn.restype)
            assert fn.argtypes is not None, f"{name}: argtypes not set"
            assert list(fn.argtypes) == [_ctype(nat, p) for p in params], (name, params, fn.argtypes)


def test_bad_arguments_return_error_string(nat):
    L = nat.lib()
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    rc = L.ba_fwd_chunk(z4, z4, z4, z4, zr, z4, 1, 128, 128, 1, 96, 1.0, 0, 0, 3, 1, None)
    assert rc != 0 and b"head dim" in L.ba_last_error()
    rc = L.ba_fwd_chunk(z4, z4, z4, z4, zr, z4, 1, 128, 128, 1, 128, 1.0, 0, 0, 3, 1, None)
    assert rc != 0 and b"null" in L.ba_last_error()
    rc = L.ba_ring_post(None, None, None, None, 0, None)
    assert rc != 0
    rc = L.ba_ring_arena_create(None, 1 << 20, None, None)
    assert rc != 0 and b"ba_ring_arena_create" in L.ba_last_error()
    rc = L.ba_ring_arena_connect(None, None, None)
    assert rc != 0 and b"ba_ring_arena_connect" in L.ba_last_error()
    assert L.ba_version() >= 200


def test_gqa_symbols_exported_and_bound(nat):
    L = ctypes.CDLL(nat.LIB_PATH)
    for name in ("ba_fwd_chunk_gqa", "ba_bwd_chunk_gqa"):
        assert hasattr(L, name), name
        assert name in nat.exported_symbols()
    assert nat.lib().ba_version() >= 201


@pytest.mark.parametrize("H,H_kv", [(32, 5), (4, 8), (8, 0), (8, -2)])
def test_bad_kv_head_count_returns_error_string(nat, H, H_kv):
    """A K/V head count that is not positive or does not divide the query head count is rejected with an error
    string naming H_kv before anything touches the GPU."""
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


def test_missing_library_fails_loudly(nat, monkeypatch):
    monkeypatch.setattr(nat, "_lib", None)
    monkeypatch.setattr(nat, "LIB_PATH", "/nonexistent/libburst_attn_b200.so")
    with pytest.raises(nat.NativeLibraryError):
        nat.lib()


def test_receive_arena_bump_allocator_is_symmetric_and_aligned():
    """Host logic of the copy-engine transport's receive arena (burst_attn/comm.py): buffers are carved in
    call order at 1 KiB-aligned offsets, so equal call sequences give equal offsets on every rank, and the
    size announced by Ring.begin covers them."""
    import torch
    from burst_attn import comm

    ring = comm._NativeRing.__new__(comm._NativeRing)  # no library / device needed for the carving logic
    ring.ce = True
    sizes = [3 * 5 * 7 * 2, 1024, 4 * 33]
    ring.arena = torch.zeros(sum(comm._align(n) for n in sizes), dtype=torch.uint8)
    ring.arena_off = 0
    a = ring.empty((3, 5, 7), torch.bfloat16)
    b = ring.empty((256,), torch.float32)
    c = ring.empty((33,), torch.float32)
    base = ring.arena.data_ptr()
    assert [t.data_ptr() - base for t in (a, b, c)] == [0, 1024, 2048]
    assert a.shape == (3, 5, 7) and a.dtype == torch.bfloat16 and c.is_contiguous()
    with pytest.raises(AssertionError):
        ring.empty((1,), torch.float32)  # beyond what begin() announced


def test_copy_engine_setup_agrees_across_ranks_and_falls_back(monkeypatch):
    """Host logic of burst_attn/comm.py around the copy-engine arena, with the C-ABI and torch.distributed faked:
    (1) success path: create -> all-gather (ok, handle) -> connect with the NEIGHBOURS' handles -> all-gather ok;
    (2) a rank whose create fails makes EVERY rank raise CopyEngineUnavailable after the same collectives;
    (3) Ring.begin turns that into a process-wide switch to NCCL when the transport was only the default, and
        re-raises when BA_RING_TRANSPORT=ce asked for it by name."""
    import torch
    from burst_attn import comm, native

    calls = []

    class FakeLib:
        def __init__(self, fail_create=False):
            self.fail_create = fail_create

        def ba_ring_arena_create(self, handle, nbytes, base_ref, hbuf):
            calls.append("create")
            if self.fail_create:
                return 2
            hbuf[0] = 7  # this rank's "handle"
            return 0

        def ba_ring_arena_connect(self, handle, prv, nxt):
            calls.append(("connect", prv[0], nxt[0]))
            return 0

        def ba_last_error(self):
            return b"no CUDA IPC here"

    world, rank = 4, 1

    def fake_all_gather(out, obj, group=None):
        calls.append("gather")
        for i in range(len(out)):
            out[i] = obj
        if isinstance(obj, tuple):  # neighbours' handles differ from ours
            out[(rank - 1) % world] = (peer_ok, bytes([3]) + obj[1][1:])
            out[(rank + 1) % world] = (True, bytes([5]) + obj[1][1:])

    class NoCtx:
        def __enter__(self): return self
        def __exit__(self, *a): return False

    monkeypatch.setattr(comm.dist, "all_gather_object", fake_all_gather)
    monkeypatch.setattr(comm.dist, "barrier", lambda group=None: calls.append("barrier"))
    monkeypatch.setattr(torch.cuda, "synchronize", lambda d=None: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: NoCtx())
    monkeypatch.setattr(torch, "as_tensor", lambda obj, device=None: torch.zeros(obj.__cuda_array_interface__["shape"], dtype=torch.uint8))
    fake = FakeLib()
    monkeypatch.setattr(native, "lib", lambda: fake)

    def mk(lib):
        r = comm._NativeRing.__new__(comm._NativeRing)
        r.lib, r.group, r.device, r.world, r.rank, r.ce = lib, None, torch.device("cpu"), world, rank, True
        r.arena, r.arena_off, r.handle = None, 0, None
        return r

    peer_ok = True
    ring = mk(fake)
    ring.begin(5000)
    assert calls == ["barrier", "create", "gather", ("connect", 3, 5), "gather", "barrier"]
    assert ring.arena is not None and ring.arena.numel() >= 5000

    calls.clear()
    peer_ok = False  # the previous rank could not create its arena: we raise too, after the same first gather
    with pytest.raises(comm.CopyEngineUnavailable):
        mk(fake).begin(5000)
    assert calls == ["barrier", "create", "gather"]

    calls.clear()
    peer_ok = True
    bad = FakeLib(fail_create=True)
    monkeypatch.setattr(native, "lib", lambda: bad)
    with pytest.raises(comm.CopyEngineUnavailable, match="no CUDA IPC here"):
        mk(bad).begin(5000)
    assert calls == ["barrier", "create", "gather"]

    # Ring.begin: default transport -> fall back to NCCL for the whole process; named transport -> re-raise
    class FailingNative:
        ce = True

        def begin(self, n):
            raise comm.CopyEngineUnavailable("x")

    like = type("T", (), {"is_cuda": True, "device": torch.device("cpu")})()
    monkeypatch.setattr(comm, "_ce_disabled", False)
    monkeypatch.delenv("BA_RING_TRANSPORT", raising=False)
    monkeypatch.setattr(comm, "get_world_size", lambda g=None: 4)
    monkeypatch.setattr(comm, "get_rank", lambda g=None: 1)
    r = comm.Ring(None, transport="ce")
    r._native = FailingNative()
    with pytest.warns(UserWarning, match="using NCCL"):
        r.begin(like, [1024])
    assert r.transport == "nccl" and r._native is None and comm._ce_disabled
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "4")
    assert comm.default_transport() == "nccl"
    monkeypatch.setattr(comm, "_ce_disabled", False)
    monkeypatch.setenv("BA_RING_TRANSPORT", "ce")
    r = comm.Ring(None)
    r._native = FailingNative()
    with pytest.raises(comm.CopyEngineUnavailable):
        r.begin(like, [1024])
