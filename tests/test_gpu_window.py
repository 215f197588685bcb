"""Sliding-window (band) attention on the GPU: the tile kernels' band mask, the flash_attn_* wrappers and the ring.

* Chunk kernels: ``NativeOps.fwd_chunk`` / ``bwd_chunk`` with a band ``("band", lo, hi)`` -- key b visible to row a iff
  a + lo <= b <= a + hi -- over chains of K/V chunks with carried state, against the fp64 oracle and the 16-bit model
  (``lowp_model``): bands inside one tile, across 128-key tiles and 64-row blocks, narrower than a warpgroup's 64
  rows, beyond Sk (dead rows), ragged Sq / Sk, head dim 64 and 128, bf16 and fp16, GQA, a key bias, carried state.
  Dead rows must give O = 0, dQ = 0 and lse = -inf exactly, keys no row sees dK = dV = 0 exactly, and deterministic
  mode must be bitwise reproducible.  Three faults of the band's lower edge injected into the model must be rejected.
* ``flash_attn_func`` / ``_kvpacked_func`` / ``_qkvpacked_func`` with ``window_size``, causal and not, Sq != Sk, with
  BA_L2_BLOCK = 256 so that rows whose first visible key block is not block 0 start their state in later launches.
* The ring at W = 2, 4 and 8 on one device (``ring_band`` over ``ring_harness``), flat and hierarchical, in all three shard layouts.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import band_oracle as bo  # noqa: E402
import lowp_band  # noqa: E402
import lowp_model as lm  # noqa: E402
import ring_band as rb  # noqa: E402
import ring_harness as rh  # noqa: E402
from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402

BF16, FP16 = torch.bfloat16, torch.float16
lowp_band.install()  # lowp_model's model, oracle chain and comparator take the band masks below


def _kw(m, bias):
    """fwd_chunk / bwd_chunk arguments of a mask: (causal, offset, extra keywords)."""
    kw = {} if bias is None else {"bias": bias}
    if m is None:
        return False, 0, kw
    if m[0] == "causal_offset":
        return True, m[1], kw
    _, lo, hi = m
    if lo is not None:
        kw["lower"] = lo
    return hi is not None, 0 if hi is None else hi, kw


def native_chain(x, det_runs=2):
    ops = NativeOps()
    q, do, ks, vs = x["q"], x["do"], x["ks"], x["vs"]
    B, Sq, H = q.shape[:3]
    n = len(ks)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    o_acc = torch.empty(q.shape, device="cuda", dtype=torch.float32) if n > 1 else None
    states = []
    for c, m in enumerate(x["masks"]):
        causal, off, kw = _kw(m, x["biases"][c])
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, x["scale"], causal, off, c == 0, c == n - 1, 1, **kw)
        if c < n - 1:
            states.append((o_acc.clone(), lse.clone()))
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, 1)

    def backward(det):
        dq = torch.zeros(q.shape, device="cuda", dtype=torch.float32)
        dks, dvs = [], []
        for c, m in enumerate(x["masks"]):
            causal, off, kw = _kw(m, x["biases"][c])
            dk = torch.zeros(ks[c].shape, device="cuda", dtype=torch.float32)
            dv = torch.zeros(vs[c].shape, device="cuda", dtype=torch.float32)
            ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, x["scale"], causal, off, 1, deterministic=det,
                          **kw)
            dks.append(dk)
            dvs.append(dv)
        return dq, dks, dvs

    dq, dks, dvs = backward(False)
    dets = [backward(True) for _ in range(det_runs)]
    torch.cuda.synchronize()
    return dict(o=out, lse=lse, states=states, dq=dq, dk=dks, dv=dvs), dets


def _case(sq, chunks, D=128, dtype=BF16, bias=None, H=2, Hkv=None, tag=""):
    """chunks: [(Sk, lo, hi)]; the case id carries the bands (it seeds the inputs)."""
    ch = "+".join(f"{sk}b{lo}_{hi}" for sk, lo, hi in chunks)
    c = lm._case(sq, [(sk, None) for sk, _, _ in chunks], D, dtype, bias=bias, H=H, Hkv=Hkv, tag=f"band_{tag}{ch}_")
    c["bands"] = [("band", lo, hi) for _, lo, hi in chunks]
    return c


CASES = [
    _case(257, [(257, -5, 0)]),                      # causal window of 6 keys: inside one tile
    _case(257, [(257, -100, 0)], 64, FP16),          # crosses 128-key tiles and 64-row blocks
    _case(383, [(383, -30, 30)]),                    # two-sided, narrower than a warpgroup's 64 rows
    _case(383, [(383, 0, 0)], 64, BF16),             # the diagonal only
    _case(255, [(513, 129, 200)], 128, FP16),        # above the diagonal, Sq != Sk
    _case(129, [(257, 200, None)]),                  # lower edge only; rows from 57 on see nothing (beyond Sk)
    _case(130, [(1, -3, 2)], 64, FP16),              # one key
    _case(65, [(300, -64, 63)], 128, BF16),          # ragged
    _case(200, [(500, 150, 290)], 128, BF16, H=4, Hkv=2),   # GQA
    _case(200, [(333, -40, 40)], 64, FP16, H=4, Hkv=1),     # MQA
    _case(257, [(257, -70, 10)], 128, BF16, bias="randn"),  # key bias with a window
    _case(129, [(257, -64, 128)], 64, FP16, bias="edge_inf"),
    # carried state: views of one windowed problem, chunk offsets shifted by the chunk's start
    _case(200, [(128, 0 - 60, 0), (128, -128 - 60, -128), (100, -256 - 60, -256)], 128, BF16, tag="chain_"),
    _case(129, [(64, 300, None), (128, -64, 0), (200, -190, -100)], 64, FP16, tag="dead1st_"),
]


def _inputs(case):
    x = lm.make_inputs(case, "cuda")
    x["masks"] = case["bands"]
    return x


def _check_dead(x, got, ref):
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)
    assert torch.equal(torch.isinf(got["lse"].cpu()) & (got["lse"].cpu() < 0), dead)
    rows = dead.permute(0, 2, 1)
    assert (got["o"].cpu()[rows] == 0).all(), "O of a row that sees nothing"
    assert (got["dq"].cpu()[rows] == 0).all(), "dQ of a row that sees nothing"
    B, Sq, H = x["q"].shape[:3]
    for c, (k, m) in enumerate(zip(x["ks"], x["masks"])):
        Sk, Hkv = k.shape[1], k.shape[2]
        seen = (~dead).unsqueeze(-1) & lowp_band.visible(Sq, Sk, m)
        if x["biases"][c] is not None:
            seen = seen & ~torch.isinf(x["biases"][c].cpu()).unsqueeze(2)
        seen = seen.any(2).view(B, Hkv, H // Hkv, Sk).any(2).permute(0, 2, 1)
        for name in ("dk", "dv"):
            assert (got[name][c].cpu()[~seen] == 0).all(), f"{name} of a key no row sees (chunk {c})"


def _absmax(x):
    return [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1], x["biases"][:c + 1])
            for c in range(len(x["ks"]))]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_band_chunks_within_model(case):
    x = _inputs(case)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got, dets = native_chain(x)
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], _absmax(x))
    _check_dead(x, got, ref)
    (dq0, dk0, dv0), (dq1, dk1, dv1) = dets
    assert torch.equal(dq0, dq1) and all(torch.equal(a, b) for a, b in zip(dk0 + dv0, dk1 + dv1)), \
        "deterministic mode is not bitwise reproducible with a band"
    lm.assert_chain_within_model(case["id"] + " deterministic", dict(got, dq=dq0, dk=dk0, dv=dv0), ref, model,
                                 case["dtype"], _absmax(x))


MUTANT_CASE = _case(383, [(383, -100, 20)], 128, BF16, tag="mutant_")


@pytest.mark.parametrize("mutant", lowp_band.BAND_MUTANTS)
def test_band_mutants_are_rejected(mutant):
    """The comparator rejects the model with a fault at the band's lower edge, on the same inputs as the kernels."""
    x = _inputs(MUTANT_CASE)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got = lm.lowp_chain(*args, mutant=mutant)
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    with pytest.raises(AssertionError):
        lm.assert_chain_within_model(mutant, got, ref, model, MUTANT_CASE["dtype"], _absmax(x))


# --------------------------------------------------------------------------- #
# the flash_attn_* wrappers
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("l2", [None, 256])
@pytest.mark.parametrize("fn", ["func", "kvpacked", "qkvpacked"])
@pytest.mark.parametrize("causal,window,sq,sk", [(True, (100, -1), 700, 700), (False, (64, 300), 700, 700),
                                                 (True, (200, 5), 333, 900), (False, (0, 0), 600, 600),
                                                 (False, (-1, 30), 900, 401)])
def test_flash_wrappers_window(monkeypatch, fn, causal, window, sq, sk, l2):
    if fn == "qkvpacked" and sq != sk:
        pytest.skip("qkvpacked has one sequence length")
    if l2:
        monkeypatch.setenv("BA_L2_BLOCK", str(l2))
    else:
        monkeypatch.delenv("BA_L2_BLOCK", raising=False)
    left, right = window
    off = sk - sq
    band = ("band", None if left < 0 else off - left, 0 + off if causal else (None if right < 0 else off + right))
    case = _case(sq, [(sk, band[1], band[2])], 128, BF16, H=4, tag=f"api_{fn}_{int(causal)}_{l2}_")
    x = _inputs(case)
    q, k, v = x["q"], x["ks"][0], x["vs"][0]
    if fn == "func":
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = flash_attn_func(qq, kk, vv, None, causal, x["scale"], window)
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), x["do"])
    elif fn == "kvpacked":
        qq, kv = q.clone().requires_grad_(), torch.stack([k, v], 2).requires_grad_()
        o = flash_attn_kvpacked_func(qq, kv, None, causal, x["scale"], window)
        dq, dkv = torch.autograd.grad(o, (qq, kv), x["do"])
        dk, dv = dkv[:, :, 0], dkv[:, :, 1]
    else:
        qkv = torch.stack([q, k, v], 2).requires_grad_()
        o = flash_attn_qkvpacked_func(qkv, None, causal, x["scale"], window)
        (dqkv,) = torch.autograd.grad(o, (qkv,), x["do"])
        dq, dk, dv = dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2]
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    lm.assert_api_within_model(case["id"], dict(o=o, dq=dq, dk=dk, dv=dv), lm.oracle_chain(*args),
                               lm.lowp_chain(*args), BF16)
    # cross-check the band against flash-attn's window convention in the dense oracle
    o_ref, _ = bo.dense_attention(q.cpu(), k.cpu(), v.cpu(), x["scale"], causal, window)
    torch.testing.assert_close(o.float().cpu(), o_ref.float(), rtol=2e-2, atol=2e-2)


# --------------------------------------------------------------------------- #
# the ring on one device
# --------------------------------------------------------------------------- #
def _ring_jobs(world):
    S = 128 if world == 8 else 192
    j = lambda *a, **kw: rb.window_job(world, *a, B=1, **kw)  # noqa: E731
    jobs = [j("none", BF16, 128, 2, S, (S // 2, S // 2)),               # spans neighbouring shards only
            j("zigzag", BF16, 128, 2, S, (S + 40, -1)),                 # spans several halves
            j("striped", FP16, 64, 4, S, (37, -1)),
            j("striped", BF16, 128, 2, S, (20, 9), causal=False),       # two-sided, non-causal striped
            j("none", FP16, 64, 1, S, (0, 0))]
    if world == 4:
        jobs += [j(m, BF16, 128, 2, S, (150, 3), intra=2, dq_groups=True) for m in ("none", "zigzag", "striped")]
        jobs += [j("zigzag", BF16, 128, 2, 320, (300, -1), l2=128, det=True)]
    if world == 8:
        jobs += [j("zigzag", BF16, 128, 2, S, (200, -1), intra=4)]
    return jobs


RING_JOBS = {w: _ring_jobs(w) for w in (2, 4, 8)}
RING_CASES = [j for w in RING_JOBS for j in RING_JOBS[w]]


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) != (9, 0):
        pytest.skip("needs an sm_90 GPU")
    return rb.WindowRuns(RING_JOBS, tmp_path_factory, timeout=900)


@pytest.mark.parametrize("job", RING_CASES, ids=lambda j: j["id"])
def test_ring_window_within_model(runs, job):
    rb.check_window_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))
