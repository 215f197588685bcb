"""The tile kernels at their edges, against a 16-bit error model (tests/lowp_model.py).

Every case of ``lowp_model.SWEEP`` runs ``NativeOps.fwd_chunk`` over a chain of K/V chunks with carried state, then
``delta`` and ``bwd_chunk`` per chunk, straight through the C-ABI, and compares each output with the fp64 oracle
scaled by the error of the rounding model on the same inputs: the fp32 (o_acc, lse) state after every non-last chunk,
O, lse, dQ, dK and dV.  The backward runs three times: once in the default mode and twice with deterministic=True;
the deterministic runs must be bitwise equal and both modes within the model.  The sweep covers Sq and Sk one either
side of the forward's 128-row / 128-key and the backward's 64-row tiles, causal offsets one key either side of every
tile edge on both signs, softmax scales 0.01 .. 1, rising / last-tile / uniform score distributions, chains of up to
16 chunks with rows that are dead in the first chunk, key biases with -inf tiles, tile-edge keys and fully masked
rows, batch-strided and [B,H,S,D] layouts, grouped-query attention and fp16 inputs scaled by 4.  The public API is
checked with caller-chosen scales through the L2-blocked driver.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import lowp_model as lm  # noqa: E402
from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402


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


def native_chain(x, layout, deterministic_runs=2):
    """The kernels on one case.  Returns (result dict like lowp_chain's, [deterministic results (dq, dk, dv)])."""
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
        kw = {} if x["biases"][c] is None else {"bias": x["biases"][c]}
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, x["scale"], m is not None, 0 if m is None else m[1],
                      c == 0, c == n - 1, sd, **kw)
        if c < n - 1:
            states.append((_logical(o_acc, layout).clone(), lse.clone()))
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, sd)

    def backward(det):
        dq = torch.zeros(q.shape, device="cuda", dtype=torch.float32)
        dks, dvs = [], []
        for c, m in enumerate(x["masks"]):
            kw = {} if x["biases"][c] is None else {"bias": x["biases"][c]}
            dk = torch.zeros(ks[c].shape, device="cuda", dtype=torch.float32)
            dv = torch.zeros(vs[c].shape, device="cuda", dtype=torch.float32)
            ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, x["scale"], m is not None,
                          0 if m is None else m[1], sd, deterministic=det, **kw)
            dks.append(_logical(dk, layout))
            dvs.append(_logical(dv, layout))
        return _logical(dq, layout), dks, dvs

    dq, dks, dvs = backward(False)
    dets = [backward(True) for _ in range(deterministic_runs)]
    torch.cuda.synchronize()
    res = dict(o=_logical(out, layout), lse=lse, states=states, dq=dq, dk=dks, dv=dvs)
    return res, dets


def _check_dead(x, got, ref):
    """Rows that see no key: O = 0, lse = -inf, dQ = 0 exactly; keys no row sees: dK = dV = 0 exactly."""
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)  # [B,H,Sq]
    if dead.any():
        rows = dead.permute(0, 2, 1)  # [B,Sq,H]
        assert (got["o"].cpu()[rows] == 0).all(), "O of a row that sees nothing"
        assert (got["dq"].cpu()[rows] == 0).all(), "dQ of a row that sees nothing"
    B, Sq, H = x["q"].shape[:3]
    alive = ~dead.cpu()  # [B,H,Sq]
    for c, (k, m) in enumerate(zip(x["ks"], x["masks"])):
        Sk, Hkv = k.shape[1], k.shape[2]
        vis = lm.visible(Sq, Sk, m)
        vis = torch.ones(Sq, Sk, dtype=torch.bool) if vis is None else vis
        seen = alive.unsqueeze(-1) & vis  # [B,H,Sq,Sk]
        if x["biases"][c] is not None:
            seen = seen & ~torch.isinf(x["biases"][c].cpu()).unsqueeze(2)
        seen = seen.any(2).view(B, Hkv, H // Hkv, Sk).any(2).permute(0, 2, 1)  # [B,Sk,Hkv]
        for name in ("dk", "dv"):
            assert (got[name][c].cpu()[~seen] == 0).all(), f"{name} of a key no row sees (chunk {c})"


@pytest.mark.parametrize("case", lm.SWEEP, ids=[c["id"] for c in lm.SWEEP])
def test_tile_edges_within_model(case):
    x = lm.make_inputs(case, "cuda")
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got, dets = native_chain(x, case["layout"])
    model = lm.lowp_chain(*args)
    ref = lm.oracle_chain(*args)
    n = len(x["ks"])
    absmax = [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1], x["biases"][:c + 1])
              for c in range(n)]
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)
    _check_dead(x, got, ref)
    # deterministic mode: bitwise reproducible, and within the model as well
    (dq0, dk0, dv0), (dq1, dk1, dv1) = dets
    assert torch.equal(dq0, dq1) and all(torch.equal(a, b) for a, b in zip(dk0 + dv0, dk1 + dv1))
    got_det = dict(got, dq=dq0, dk=dk0, dv=dv0)
    lm.assert_chain_within_model(case["id"] + " deterministic", got_det, ref, model, case["dtype"], absmax)
    if case["dist"] == "zero_q" and case["bias"] is None:  # uniform attention, in closed form
        H = case["H"]
        o_cf, lse_cf = lm.uniform_closed_form([lm._kv_heads(v.cpu(), H) for v in x["vs"]], x["masks"], case["sq"])
        lm.assert_within_model(f"o_closed_form[{case['id']}]", got["o"], o_cf, model["o"], case["dtype"])
        lm.assert_lse(f"lse_closed_form[{case['id']}]", got["lse"], lse_cf.view(1, 1, -1).expand_as(got["lse"]),
                      torch.zeros_like(got["lse"]).cpu())


# the public API with a caller-chosen softmax_scale; a small BA_L2_BLOCK splits every call into sub-launches with
# causal offsets, which must all carry the caller's scale
@pytest.mark.parametrize("striped", [False, True])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("scale,D,dtype,S", [(0.05, 128, torch.bfloat16, 600), (1.0, 64, torch.float16, 334),
                                             (1.0, 128, torch.bfloat16, 258)])
def test_public_api_softmax_scale(monkeypatch, striped, causal, scale, D, dtype, S):
    monkeypatch.setenv("BA_L2_BLOCK", "128")
    case = lm._case(S, [(S, 0 if causal else None)], D, dtype, scale=scale, tag="api_")
    x = lm.make_inputs(case, "cuda")
    q, k, v = (t.clone().requires_grad_() for t in (x["q"], x["ks"][0], x["vs"][0]))
    fn = burst_attn_func_striped if striped else burst_attn_func
    o = fn(q, k, v, scale, "cuda", causal)
    dq, dk, dv = torch.autograd.grad(o, (q, k, v), x["do"])
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    model = lm.lowp_chain(*args)
    ref = lm.oracle_chain(*args)
    name = f"{case['id']}_{'striped' if striped else 'contiguous'}"
    lm.assert_api_within_model(name, dict(o=o, dq=dq, dk=dk, dv=dv), ref, model, dtype)


def test_report_worst_ratios():
    """Runs last: prints the worst error / bound seen per output and dtype (the constants keep these <= 0.5)."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(lm.WORST.items()):
        print(f"worst {name:>22s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
