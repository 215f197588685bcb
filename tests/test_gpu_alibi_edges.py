"""The ALiBi tile kernels at their edges, against the 16-bit error model (tests/lowp_alibi.py).

Every case of ``lowp_alibi.ALIBI_SWEEP`` runs ``NativeOps.fwd_chunk`` with ``alibi=(slopes, dist0, pstride)`` over a
chain of K/V chunks with carried state, then ``delta`` and ``bwd_chunk`` per chunk, straight through the C-ABI, and
compares each output with the fp64 ALiBi oracle scaled by the error of the rounding model on the same inputs: the
fp32 (o_acc, lse) state after every non-last chunk, O, lse, dQ, dK and dV, per (b, s, h) row.  The backward runs once
in the default mode and twice with deterministic=True (bitwise equal, and within the model).  Rows that see nothing
must give O = 0, dQ = 0 and lse = -inf exactly, keys no row sees dK = dV = 0 exactly.

The sweep puts tiles of 64 rows x 128 keys on every sign edge (dmin in {0, -1, -pstride}, dmax in {0, 1, pstride})
at pstride 1, 2, 3, 4 and 8, with causal offsets and band lower edges on them; chains near -> far, far -> near,
far -> far and of 16 chunks at slopes 0.5 .. 1; |dist0| above 2^24; standard, tiny, zero, negative and per-(batch,
head) slopes; GQA with a slope per query head; head dim 64 and 128, bf16 and fp16, and the flash, [B,H,S,D] and
batch-strided layouts.  Every fault of ``ALIBI_MUTANTS`` injected into the model is rejected on the same inputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import lowp_alibi as la  # noqa: E402
import lowp_model as lm  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402

_BY_ID = {c["id"]: c for c in la.ALIBI_SWEEP}


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


def _kw(m):
    """fwd_chunk / bwd_chunk arguments of a mask: (causal, offset, lower)."""
    if m is None:
        return False, 0, None
    if m[0] == "causal_offset":
        return True, m[1], None
    _, lo, hi = m
    return hi is not None, 0 if hi is None else hi, lo


def native_chain(x, layout, det_runs=2):
    """The ALiBi kernels on one case: (result dict like lowp_model.lowp_chain's, [deterministic (dq, dks, dvs)])."""
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
        causal, off, lower = _kw(m)
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, x["scale"], causal, off, c == 0, c == n - 1, sd,
                      lower=lower, alibi=x["alibis"][c])
        if c < n - 1:
            states.append((_logical(o_acc, layout).clone(), lse.clone()))
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, sd)

    def backward(det):
        dq = torch.zeros(q.shape, device="cuda", dtype=torch.float32)
        dks, dvs = [], []
        for c, m in enumerate(x["masks"]):
            causal, off, lower = _kw(m)
            dk = torch.zeros(ks[c].shape, device="cuda", dtype=torch.float32)
            dv = torch.zeros(vs[c].shape, device="cuda", dtype=torch.float32)
            ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, x["scale"], causal, off, sd, deterministic=det,
                          lower=lower, alibi=x["alibis"][c])
            dks.append(_logical(dk, layout))
            dvs.append(_logical(dv, layout))
        return _logical(dq, layout), dks, dvs

    dq, dks, dvs = backward(False)
    dets = [backward(True) for _ in range(det_runs)]
    torch.cuda.synchronize()
    return dict(o=_logical(out, layout), lse=lse, states=states, dq=dq, dk=dks, dv=dvs), dets


def _check_dead(x, got, ref):
    """Rows that see no key: O = 0, lse = -inf, dQ = 0 exactly; keys no row sees: dK = dV = 0 exactly."""
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)  # [B,H,Sq]
    assert torch.equal(torch.isinf(got["lse"].cpu()) & (got["lse"].cpu() < 0), dead)
    rows = dead.permute(0, 2, 1)
    assert (got["o"].cpu()[rows] == 0).all(), "O of a row that sees nothing"
    assert (got["dq"].cpu()[rows] == 0).all(), "dQ of a row that sees nothing"
    B, Sq, H = x["q"].shape[:3]
    for c, (k, m) in enumerate(zip(x["ks"], x["masks"])):
        Sk, Hkv = k.shape[1], k.shape[2]
        vis = lm.visible(Sq, Sk, m)
        vis = torch.ones(Sq, Sk, dtype=torch.bool) if vis is None else vis
        seen = ((~dead).unsqueeze(-1) & vis).any(2).view(B, Hkv, H // Hkv, Sk).any(2).permute(0, 2, 1)
        for name in ("dk", "dv"):
            assert (got[name][c].cpu()[~seen] == 0).all(), f"{name} of a key no row sees (chunk {c})"


def _args(x):
    return (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"])


@pytest.mark.parametrize("case", la.ALIBI_SWEEP, ids=[c["id"] for c in la.ALIBI_SWEEP])
def test_alibi_edges_within_model(case):
    x = la.make_alibi_inputs(case, "cuda")
    got, dets = native_chain(x, case["layout"])
    # the model's backward reads the kernels' lse (lowp_model.lowp_chain); lse itself is held to the oracle below
    model = lm.lowp_chain(*_args(x), alibis=x["alibis"], lse_bwd=got["lse"])
    ref = lm.oracle_chain(*_args(x), alibis=x["alibis"])
    absmax = la.absmax_prefix(x["q"], x["ks"], x["scale"], x["masks"], x["alibis"])
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)
    _check_dead(x, got, ref)
    (dq0, dk0, dv0), (dq1, dk1, dv1) = dets
    assert torch.equal(dq0, dq1) and all(torch.equal(a, b) for a, b in zip(dk0 + dv0, dk1 + dv1)), \
        "deterministic mode is not bitwise reproducible with ALiBi"
    lm.assert_chain_within_model(case["id"] + " deterministic", dict(got, dq=dq0, dk=dk0, dv=dv0), ref, model,
                                 case["dtype"], absmax)


@pytest.mark.parametrize("mutant,case_id", [(m, i) for m in la.ALIBI_MUTANTS for i in la.MUTANT_CASES[m]],
                         ids=[f"{m}-{'bf16' if 'bf16' in i else 'fp16'}" for m in la.ALIBI_MUTANTS
                              for i in la.MUTANT_CASES[m]])
def test_alibi_mutant_is_rejected(mutant, case_id):
    """The comparator rejects the model with the fault, on the kernels' inputs and device."""
    x = la.make_alibi_inputs(_BY_ID[case_id], "cuda")
    got = lm.lowp_chain(*_args(x), mutant=mutant, alibis=x["alibis"])
    model, ref = lm.lowp_chain(*_args(x), alibis=x["alibis"]), lm.oracle_chain(*_args(x), alibis=x["alibis"])
    absmax = la.absmax_prefix(x["q"], x["ks"], x["scale"], x["masks"], x["alibis"])
    worst = dict(lm.WORST)  # the rejected runs stay out of the report of the kernels' worst ratios
    try:
        with pytest.raises(AssertionError):
            lm.assert_chain_within_model(mutant, got, ref, model, _BY_ID[case_id]["dtype"], absmax)
    finally:
        lm.WORST.clear()
        lm.WORST.update(worst)


def test_report_worst_ratios():
    """Runs last: prints the worst error / bound seen per output and dtype (the constants keep these <= 0.5)."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(lm.WORST.items()):
        print(f"worst {name:>22s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
