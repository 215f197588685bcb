"""Sliding-window (band) attention on the GPU: the tile kernels' band mask, the flash_attn_* wrappers and the ring.

* Chunk kernels: every case of ``lowp_band.BAND_SWEEP`` runs ``NativeOps.fwd_chunk`` / ``bwd_chunk`` with a band
  ``("band", lo, hi)`` -- key b visible to row a iff a + lo <= b <= a + hi -- over a chain of K/V chunks with carried
  state, straight through the C-ABI, against the fp64 oracle scaled by the error of the 16-bit model (``lowp_model``):
  the fp32 (o_acc, lse) state after every non-last chunk, O, lse, dQ, dK and dV per (b, s, h) row.  The sweep puts the
  band's lower edge on every phase of the forward's 128-key tiles and warpgroups and on the backward's i_end and
  need_lo boundaries, reaches CTAs and key blocks with no work, the host's lower-edge clamps, the deterministic mode's
  turn counters from a key block x_min >= 1, chains of up to 16 chunks with rows dead, revived and blind in the last
  chunk, key biases that mask the band's edge or all of it, ragged Sq / Sk, head dim 64 and 128, bf16 and fp16, GQA
  and MQA, and the flash, [B,H,S,D] and batch-strided layouts.  Dead rows must give O = 0, dQ = 0 and lse = -inf
  exactly, keys no row sees dK = dV = 0 exactly, and deterministic mode must be bitwise reproducible.  Every fault of
  ``lowp_band.BAND_MUTANTS`` injected into the model is rejected on the same inputs.
* Causal offsets at the ends of the C-ABI's int range give what the nearest in-range offsets (Sk, -Sq) give.
* ``flash_attn_func`` / ``_kvpacked_func`` / ``_qkvpacked_func`` with ``window_size``, causal and not, Sq != Sk, with
  BA_L2_BLOCK = 256 so that rows whose first visible key block is not block 0 start their state in later launches.
* The ring at W = 2, 4 and 8 on one device (``ring_harness``), flat and hierarchical, in all three shard layouts.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import lowp_band  # noqa: E402
import lowp_model as lm  # noqa: E402
import mask_oracle as mo  # noqa: E402
import ring_harness as rh  # noqa: E402
from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402

BF16, FP16 = torch.bfloat16, torch.float16
_BY_ID = {c["id"]: c for c in lowp_band.BAND_SWEEP}


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


def _kernel_layout(t, layout):
    """A view of the logical [B,S,H,D] tensor t as the kernels see it in this case (values unchanged)."""
    if layout == "normal":
        return t.transpose(1, 2).contiguous()  # [B,H,S,D] storage
    if layout == "bstride":
        big = torch.zeros((2 * t.shape[0],) + tuple(t.shape[1:]), device=t.device, dtype=t.dtype)
        big[::2] = t
        return big[::2]
    return t


def _logical(t, layout):
    return t.transpose(1, 2) if layout == "normal" else t


def native_chain(x, layout="flash", det_runs=2):
    """The band kernels on one case: (result dict like lowp_chain's, [deterministic (dq, dks, dvs)])."""
    ops = NativeOps()
    sd = 2 if layout == "normal" else 1
    q, do = _kernel_layout(x["q"], layout), _kernel_layout(x["do"], layout)
    ks = [_kernel_layout(k, layout) for k in x["ks"]]
    vs = [_kernel_layout(v, layout) for v in x["vs"]]
    B, Sq, H = x["q"].shape[:3]
    n = len(ks)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    o_acc = torch.empty(q.shape, device="cuda", dtype=torch.float32) if n > 1 else None
    states = []
    for c, m in enumerate(x["masks"]):
        causal, off, kw = _kw(m, x["biases"][c])
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, x["scale"], causal, off, c == 0, c == n - 1, sd, **kw)
        if c < n - 1:
            states.append((_logical(o_acc, layout).clone(), lse.clone()))
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, sd)

    def backward(det):
        dq = torch.zeros(q.shape, device="cuda", dtype=torch.float32)
        dks, dvs = [], []
        for c, m in enumerate(x["masks"]):
            causal, off, kw = _kw(m, x["biases"][c])
            dk = torch.zeros(ks[c].shape, device="cuda", dtype=torch.float32)
            dv = torch.zeros(vs[c].shape, device="cuda", dtype=torch.float32)
            ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, x["scale"], causal, off, sd, deterministic=det,
                          **kw)
            dks.append(_logical(dk, layout))
            dvs.append(_logical(dv, layout))
        return _logical(dq, layout), dks, dvs

    dq, dks, dvs = backward(False)
    dets = [backward(True) for _ in range(det_runs)]
    torch.cuda.synchronize()
    return dict(o=_logical(out, layout), lse=lse, states=states, dq=dq, dk=dks, dv=dvs), dets


def _check_dead(x, got, ref):
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)
    assert torch.equal(torch.isinf(got["lse"].cpu()) & (got["lse"].cpu() < 0), dead)
    rows = dead.permute(0, 2, 1)
    assert (got["o"].cpu()[rows] == 0).all(), "O of a row that sees nothing"
    assert (got["dq"].cpu()[rows] == 0).all(), "dQ of a row that sees nothing"
    B, Sq, H = x["q"].shape[:3]
    for c, (k, m) in enumerate(zip(x["ks"], x["masks"])):
        Sk, Hkv = k.shape[1], k.shape[2]
        seen = (~dead).unsqueeze(-1) & lm.visible(Sq, Sk, m)
        if x["biases"][c] is not None:
            seen = seen & ~torch.isinf(x["biases"][c].cpu()).unsqueeze(2)
        seen = seen.any(2).view(B, Hkv, H // Hkv, Sk).any(2).permute(0, 2, 1)
        for name in ("dk", "dv"):
            assert (got[name][c].cpu()[~seen] == 0).all(), f"{name} of a key no row sees (chunk {c})"


def _absmax(x):
    return [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1], x["biases"][:c + 1])
            for c in range(len(x["ks"]))]


def _args(x):
    return (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])


def _check_chain(name, x, got, dets, dtype, model=None, ref=None):
    """got / dets of native_chain within the model, dead rows and unseen keys exact, deterministic runs bitwise equal
    and within the model."""
    model = lm.lowp_chain(*_args(x)) if model is None else model
    ref = lm.oracle_chain(*_args(x)) if ref is None else ref
    lm.assert_chain_within_model(name, got, ref, model, dtype, _absmax(x))
    _check_dead(x, got, ref)
    (dq0, dk0, dv0), (dq1, dk1, dv1) = dets
    assert torch.equal(dq0, dq1) and all(torch.equal(a, b) for a, b in zip(dk0 + dv0, dk1 + dv1)), \
        "deterministic mode is not bitwise reproducible with a band"
    lm.assert_chain_within_model(name + " deterministic", dict(got, dq=dq0, dk=dk0, dv=dv0), ref, model, dtype,
                                 _absmax(x))


@pytest.mark.parametrize("case", lowp_band.BAND_SWEEP, ids=[c["id"] for c in lowp_band.BAND_SWEEP])
def test_band_chunks_within_model(case):
    x = lowp_band.make_band_inputs(case, "cuda")
    got, dets = native_chain(x, case["layout"])
    _check_chain(case["id"], x, got, dets, case["dtype"])


@pytest.mark.parametrize("mutant,case_id", [(m, i) for m in lowp_band.BAND_MUTANTS for i in lowp_band.MUTANT_CASES[m]],
                         ids=[f"{m}-{'bf16' if 'bf16' in i else 'fp16'}" for m in lowp_band.BAND_MUTANTS
                              for i in lowp_band.MUTANT_CASES[m]])
def test_band_mutants_are_rejected(mutant, case_id):
    """The comparator rejects the model with a fault of the band, on the kernels' inputs and device."""
    case = _BY_ID[case_id]
    x = lowp_band.make_band_inputs(case, "cuda")
    got = lm.lowp_chain(*_args(x), mutant=mutant)
    model, ref = lm.lowp_chain(*_args(x)), lm.oracle_chain(*_args(x))
    worst = dict(lm.WORST)  # the rejected runs stay out of the report of the kernels' worst ratios
    try:
        with pytest.raises(AssertionError):
            lm.assert_chain_within_model(mutant, got, ref, model, case["dtype"], _absmax(x))
    finally:
        lm.WORST.clear()
        lm.WORST.update(worst)


# --------------------------------------------------------------------------- #
# causal offsets at the ends of the C-ABI's int range
# --------------------------------------------------------------------------- #
# The C-ABI takes any int causal_offset (key j visible to row i iff j <= i + causal_offset); an offset >= Sk - 1 shows
# every key and one <= -Sq none, so each chain must compute bitwise what it computes with Sk and -Sq in their place.
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31
OFFSET_CASES = [
    lowp_band.bcase(257, [(383, None, I32_MAX)], 128, BF16, tag="offmax_"),
    lowp_band.bcase(257, [(383, -100, I32_MAX)], 64, FP16, tag="offmax_"),
    lowp_band.bcase(200, [(257, -60, 40), (128, None, I32_MIN), (129, -300, 300)], 128, FP16, tag="offmin_"),
    lowp_band.bcase(129, [(128, None, 0), (257, None, I32_MIN + 5), (64, -10, I32_MAX)], 64, BF16, tag="offmin_"),
]


def _in_range(masks, sq, sks):
    """The masks with every causal offset clamped into [-Sq, Sk]."""
    return [("band", lo, None if hi is None else min(max(hi, -sq), sk)) for (_, lo, hi), sk in zip(masks, sks)]


@pytest.mark.parametrize("case", OFFSET_CASES, ids=[c["id"] for c in OFFSET_CASES])
def test_causal_offset_at_int_range_ends(case):
    x = lowp_band.make_band_inputs(case, "cuda")
    y = dict(x, masks=_in_range(x["masks"], case["sq"], [k.shape[1] for k in x["ks"]]))
    got, dets = native_chain(x)
    want, want_dets = native_chain(y)
    for name in ("o", "lse"):
        assert torch.equal(got[name], want[name]), f"{name} differs from the chain with in-range offsets"
    for c, (g, w) in enumerate(zip(got["states"], want["states"])):
        assert torch.equal(g[0], w[0]) and torch.equal(g[1], w[1]), f"the state after chunk {c} differs"
    (dq, dks, dvs), (wq, wks, wvs) = dets[0], want_dets[0]
    assert torch.equal(dq, wq), "deterministic dQ differs from the chain with in-range offsets"
    for c, (a, b, e, f) in enumerate(zip(dks, wks, dvs, wvs)):
        assert torch.equal(a, b) and torch.equal(e, f), f"deterministic dK / dV of chunk {c} differ"
    _check_chain(case["id"], x, got, dets, case["dtype"])


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
    case = lowp_band.bcase(sq, [(sk, band[1], band[2])], 128, BF16, H=4, tag=f"api_{fn}_{int(causal)}_{l2}_")
    x = lowp_band.make_band_inputs(case, "cuda")
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
    o_ref, _ = mo.dense_attention(q.cpu(), k.cpu(), v.cpu(), x["scale"], causal, window)
    torch.testing.assert_close(o.float().cpu(), o_ref.float(), rtol=2e-2, atol=2e-2)


# --------------------------------------------------------------------------- #
# the ring on one device
# --------------------------------------------------------------------------- #
def _ring_jobs(world):
    S = 128 if world == 8 else 192

    def j(mode, dt, D, Hkv, S_local, window, **kw):
        return rh.ring_job(world, mode, dt, D, Hkv, S_local, B=1, window=window, **kw)

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
    return rh.WorldRuns(RING_JOBS, "native", tmp_path_factory, timeout=900)


@pytest.mark.parametrize("job", RING_CASES, ids=lambda j: j["id"])
def test_ring_window_within_model(runs, job):
    rh.check_ring_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))


def test_report_worst_ratios():
    """Runs last: prints the worst error / bound seen per output and dtype (the constants keep these <= 0.5)."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(lm.WORST.items()):
        print(f"worst {name:>22s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
