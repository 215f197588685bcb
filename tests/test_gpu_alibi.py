"""ALiBi (``alibi_slopes``) on the GPU: the tile kernels, the flash_attn_* wrappers and burst_attn_func at W = 1.

The truth is an fp64 dense attention over explicit full-sequence positions (``_ref``): row i and key j get
``-slope[b, h] |pos_q(i) - pos_k(j)|``.  Outputs must lie within a relative error of a few 16-bit unit roundoffs of
it, and each realistic fault -- the bias one position off, the absolute value dropped, the slope taken from the K/V
head under GQA, the bias formed from absolute fp32 positions -- must move the truth by more than that bound, so the
same check would reject a kernel with that fault.
"""
import math
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402
from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func  # noqa: E402

BF16, FP16 = torch.bfloat16, torch.float16
U = {BF16: 2.0 ** -8, FP16: 2.0 ** -11}


def std_slopes(H):
    """flash-attn's standard slopes 2^(-8 (h + 1) / H)."""
    return torch.tensor([2.0 ** (-8.0 * (h + 1) / H) for h in range(H)], dtype=torch.float32)


def _bias(slopes, pos_q, pos_k, fault=None):
    """fp64 [B, H, Sq, Sk] ALiBi; ``fault`` injects one kernel fault."""
    d = pos_q.double().view(-1, 1) - pos_k.double().view(1, -1)
    if fault == "off_by_one":
        d = d + 1
    a = d if fault == "no_abs" else d.abs()
    s = slopes.double()
    if fault == "abs_fp32_positions":  # slope pos_q - slope pos_k, each rounded to fp32
        sq = (slopes.float().view(*slopes.shape, 1) * pos_q.float().view(1, -1)).double()
        sk = (slopes.float().view(*slopes.shape, 1) * pos_k.float().view(1, -1)).double()
        return -(sq.unsqueeze(-1) - sk.unsqueeze(-2)).abs()
    return -s.view(*s.shape, 1, 1) * a


def _ref(q, k, v, do, scale, slopes, pos_q, pos_k, causal=False, window=None, fault=None):
    """fp64 attention on the CPU over [B, S, H, D] inputs; slopes [B, H].  Returns o, lse, dq, dk, dv."""
    q, k, v, do = (t.detach().cpu().double().requires_grad_(t is not do) for t in (q, k, v, do))
    B, Sq, H, D = q.shape
    G = H // k.shape[2]
    sl = slopes.detach().cpu()
    if fault == "gqa_kv_head":
        sl = sl[:, (torch.arange(H) // G) * G]
    kk, vv = k.repeat_interleave(G, 2), v.repeat_interleave(G, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, kk) * scale + _bias(sl, pos_q, pos_k, fault)
    d = pos_q.double().view(-1, 1) - pos_k.double().view(1, -1)
    vis = torch.ones_like(d, dtype=torch.bool)
    if causal:
        vis &= d >= 0
    if window is not None:
        left, right = window
        if left >= 0:
            vis &= d <= left
        if right >= 0:
            vis &= d >= -right
    s = s.masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse).unsqueeze(-1))
    p = torch.where(torch.isinf(lse).unsqueeze(-1), torch.zeros_like(p), p)
    o = torch.einsum("bhqk,bkhd->bqhd", p, vv)
    dq, dk, dv = torch.autograd.grad(o, (q, k, v), do)
    return o.detach(), lse.detach(), dq, dk, dv


def _rel(got, ref):
    ref = ref.double()
    return float((got.detach().cpu().double() - ref).norm() / ref.norm().clamp(min=1e-30))


def _check(name, got, ref, dtype, k_u):
    e = _rel(got, ref)
    assert e <= k_u * U[dtype], f"{name}: relative error {e:.3e} > {k_u} u = {k_u * U[dtype]:.3e}"


def _rand(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(dtype).cuda()


def _slopes(B, H, per_batch, seed):
    if not per_batch:
        return std_slopes(H).cuda(), std_slopes(H).view(1, H).expand(B, H)
    g = torch.Generator().manual_seed(seed)
    s = std_slopes(H).view(1, H) * (0.5 + torch.rand(B, H, generator=g))
    return s.cuda(), s


# (Sq, Sk, D, dtype, causal, window, H, Hkv, B, per-batch slopes)
WRAPPER_CASES = [
    (256, 256, 128, BF16, True, None, 4, 4, 1, False),
    (256, 256, 64, FP16, False, None, 4, 4, 1, False),
    (200, 333, 64, FP16, False, None, 4, 2, 2, True),
    (333, 200, 128, BF16, True, None, 4, 1, 1, False),   # rows 0..132 see no key: dead rows
    (129, 517, 128, BF16, True, (100, -1), 4, 4, 1, False),
    (300, 300, 128, FP16, False, (64, 32), 8, 2, 1, True),
    (65, 191, 96, BF16, False, None, 4, 4, 1, False),    # head dim padded up to 128
    (1000, 1200, 64, BF16, True, None, 4, 4, 1, False),
    (1000, 1200, 128, BF16, False, (300, 200), 4, 2, 1, False),
]


def _wrapper_id(c):
    sq, sk, D, dt, causal, win, H, Hkv, B, pb = c
    return (f"q{sq}_k{sk}_d{D}_{'bf16' if dt == BF16 else 'fp16'}_{'causal' if causal else 'full'}"
            f"{'' if win is None else f'_w{win[0]}.{win[1]}'}_H{H}kv{Hkv}_B{B}{'_bh' if pb else ''}")


@pytest.mark.parametrize("l2_block", [None, 256])
@pytest.mark.parametrize("case", WRAPPER_CASES, ids=_wrapper_id)
def test_flash_attn_func_alibi(case, l2_block, monkeypatch):
    Sq, Sk, D, dt, causal, win, H, Hkv, B, per_batch = case
    if l2_block is not None:
        monkeypatch.setenv("BA_L2_BLOCK", str(l2_block))
    seed = zlib.crc32(_wrapper_id(case).encode()) % 1000
    q, do = _rand((B, Sq, H, D), dt, seed), _rand((B, Sq, H, D), dt, seed + 1)
    k, v = _rand((B, Sk, Hkv, D), dt, seed + 2), _rand((B, Sk, Hkv, D), dt, seed + 3)
    slopes, sl_cpu = _slopes(B, H, per_batch, seed)
    scale = D ** -0.5
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = flash_attn_func(qq, kk, vv, None, causal, None, (-1, -1) if win is None else win, slopes)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    pos_q, pos_k = torch.arange(Sq) + Sk - Sq, torch.arange(Sk)
    ref = _ref(q, k, v, do, scale, sl_cpu, pos_q, pos_k, causal, win)
    for name, got, r, ku in (("o", o, ref[0], 2), ("dq", dq, ref[2], 4), ("dk", dk, ref[3], 4), ("dv", dv, ref[4], 4)):
        _check(name, got, r, dt, ku)
    dead = torch.isinf(ref[1]).all(0).all(0)  # rows that see no key in any batch / head
    if dead.any():
        assert (o[:, dead] == 0).all() and (dq[:, dead] == 0).all()
    # each fault moves the truth by more than the bound (the check above would reject it).  Under causal every
    # visible pair has d >= 0, so a distance one off, or without its absolute value, shifts a row's biases alike and
    # the softmax does not see it in one launch; the ring tests cover it across launches.
    faults = ([] if causal else ["off_by_one", "no_abs"]) + (["gqa_kv_head"] if Hkv < H else [])
    for f in faults:
        bad = _ref(q, k, v, do, scale, sl_cpu, pos_q, pos_k, causal, win, fault=f)
        worst = max(_rel(bad[0], ref[0]) / (2 * U[dt]), max(_rel(bad[i], ref[i]) / (4 * U[dt]) for i in (2, 3, 4)))
        assert worst > 1.5, f"fault {f} stays within the bound ({worst:.2f})"


def test_packed_wrappers_alibi():
    B, S, H, D, dt = 1, 300, 4, 64, BF16
    qkv = _rand((B, S, 3, H, D), dt, 7)
    do = _rand((B, S, H, D), dt, 8)
    slopes, sl_cpu = _slopes(B, H, False, 0)
    pos = torch.arange(S)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    ref = _ref(q, k, v, do, D ** -0.5, sl_cpu, pos, pos, True)
    x = qkv.clone().requires_grad_()
    o = flash_attn_qkvpacked_func(x, None, True, None, (-1, -1), slopes)
    (g,) = torch.autograd.grad(o, x, do)
    _check("o", o, ref[0], dt, 2)
    for i, name in enumerate(("dq", "dk", "dv")):
        _check(name, g[:, :, i], ref[2 + i], dt, 4)
    qq, kv = q.clone().requires_grad_(), qkv[:, :, 1:].clone().requires_grad_()
    o = flash_attn_kvpacked_func(qq, kv, None, True, None, (-1, -1), slopes)
    dq, dkv = torch.autograd.grad(o, (qq, kv), do)
    _check("o", o, ref[0], dt, 2)
    _check("dq", dq, ref[2], dt, 4)
    _check("dk", dkv[:, :, 0], ref[3], dt, 4)


@pytest.mark.parametrize("striped", [False, True])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("flash", ["cuda", None])
def test_burst_attn_func_alibi_one_rank(flash, causal, striped):
    if causal and flash is None:
        pytest.skip("causal attention runs in the flash layout only")
    B, S, H, Hkv, D, dt = 2, 512, 4, 2, 128, BF16
    q, do = _rand((B, S, H, D), dt, 11), _rand((B, S, H, D), dt, 12)
    k, v = _rand((B, S, Hkv, D), dt, 13), _rand((B, S, Hkv, D), dt, 14)
    slopes, sl_cpu = _slopes(B, H, True, 3)
    pos = torch.arange(S)
    ref = _ref(q, k, v, do, D ** -0.5, sl_cpu, pos, pos, causal)
    fn = burst_attn_func_striped if striped else burst_attn_func
    lay = (lambda t: t) if flash else (lambda t: t.transpose(1, 2).contiguous())
    qq, kk, vv = (lay(t).clone().requires_grad_() for t in (q, k, v))
    outs = []
    for _ in range(2):
        o = fn(qq, kk, vv, None, flash, causal, False, True, None, [None, None], (-1, -1), slopes)
        outs.append((o,) + torch.autograd.grad(o, (qq, kk, vv), lay(do)))
    for a, b in zip(*outs):  # deterministic mode: bitwise reproducible
        assert torch.equal(a, b)
    back = (lambda t: t) if flash else (lambda t: t.transpose(1, 2))
    o, dq, dk, dv = (back(t) for t in outs[0])
    _check("o", o, ref[0], dt, 2)
    for name, got, r in (("dq", dq, ref[2]), ("dk", dk, ref[3]), ("dv", dv, ref[4])):
        _check(name, got, r, dt, 4)


@pytest.mark.parametrize("dist0,pstride,slope", [(3_000_000, 1, 0.5), (-3_000_017, 1, 0.37),
                                                 (3_000_000, 3, 0.5), (-2_999_999, 2, 0.5)])
@pytest.mark.parametrize("D", [64, 128])
def test_chunk_alibi_large_positions(dist0, pstride, slope, D):
    """One forward chunk whose rows sit millions of positions from its keys (dist0 ~ 3e6): O must stay within the
    bound, and so must lse relative to its size, while a bias formed from absolute fp32 positions moves O beyond it."""
    ops = NativeOps()
    B, Sq, Sk, H, dt = 1, 200, 300, 2, BF16
    q, do = _rand((B, Sq, H, D), dt, 21), _rand((B, Sq, H, D), dt, 22)
    k, v = _rand((B, Sk, H, D), dt, 23), _rand((B, Sk, H, D), dt, 24)
    sl = torch.tensor([[slope, slope * 0.7]], dtype=torch.float32)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.fwd_chunk(q, k, v, None, lse, out, D ** -0.5, False, 0, True, True, 1, alibi=(sl.cuda(), dist0, pstride))
    # positions with pos_q(i) - pos_k(j) = pstride (i - j) + dist0, the keys at 5e6 (8e6 or 2e6 for the rows)
    base = 5_000_000
    pos_k = base + pstride * torch.arange(Sk, dtype=torch.int64)
    pos_q = base + dist0 + pstride * torch.arange(Sq, dtype=torch.int64)
    ref = _ref(q, k, v, do, D ** -0.5, sl, pos_q, pos_k)
    _check("o", out, ref[0], dt, 2)
    rel_lse = float(((lse.cpu().double() - ref[1]).abs() / (1 + ref[1].abs())).max())
    assert rel_lse <= 2.0 ** -20, rel_lse
    bad = _ref(q, k, v, do, D ** -0.5, sl, pos_q, pos_k, fault="abs_fp32_positions")
    assert _rel(bad[0], ref[0]) > 3 * U[dt], "absolute fp32 positions stay within the bound"


def test_alibi_argument_errors():
    q = torch.zeros(1, 128, 4, 64, dtype=BF16, device="cuda")
    good = std_slopes(4).cuda()
    for bad, exc in ((good.double(), TypeError), (good.cpu(), ValueError), (good[:3], ValueError),
                     (good.view(1, 1, 4), ValueError), (torch.full((4,), float("nan"), device="cuda"), ValueError)):
        with pytest.raises(exc, match="alibi_slopes"):
            flash_attn_func(q, q, q, None, False, None, (-1, -1), bad)
        with pytest.raises(exc, match="alibi_slopes"):
            burst_attn_func(q, q, q, None, "cuda", False, False, False, None, [None, None], (-1, -1), bad)
    bias = torch.zeros(1, 4, 1, 128, device="cuda")
    with pytest.raises(NotImplementedError, match="alibi_slopes"):
        flash_attn_func(q, q, q, bias, False, None, (-1, -1), good)


def test_alibi_none_is_todays_call():
    """alibi_slopes=None gives bitwise the same results as a call without the argument."""
    q, k, v, do = (_rand((1, 384, 4, 128), BF16, 30 + i) for i in range(4))
    res = []
    for extra in ((), (None,)):
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = flash_attn_func(qq, kk, vv, None, True, None, (-1, -1), *extra)
        res.append((o,) + torch.autograd.grad(o, (qq, kk, vv), do))
    for a, b in zip(*res):
        assert torch.equal(a, b)
    assert math.isfinite(float(res[0][0].detach().float().sum()))


# --------------------------------------------------------------------------- #
# chunk chains with carried state, at large positions, and faults injected into one kernel
# --------------------------------------------------------------------------- #
import lowp_model as lm  # noqa: E402
import ring_harness as rh  # noqa: E402


def _native_chain(q, ks, vs, do, scale, chunks, slopes, fwd_alibi=None, bwd_alibi=None, det=False):
    """Forward over the chunks (mask (causal, off), alibi (dist0, pstride)) with the fp32 state carried, then the
    backward of every chunk against the final (O, lse).  ``fwd_alibi`` / ``bwd_alibi``: per chunk, the (slopes,
    dist0, pstride) handed to that kernel instead of the right one (fault injection)."""
    ops = NativeOps()
    B, Sq, H = q.shape[:3]
    n = len(ks)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    o_acc = torch.empty(q.shape, device="cuda", dtype=torch.float32) if n > 1 else None
    for c, ((causal, off), (dist0, ps)) in enumerate(chunks):
        al = (fwd_alibi or {}).get(c, (slopes, dist0, ps))
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, scale, causal, off, c == 0, c == n - 1, 1, alibi=al)
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, 1)
    dq = torch.zeros(q.shape, device="cuda", dtype=torch.float32)
    dks, dvs = [], []
    for c, ((causal, off), (dist0, ps)) in enumerate(chunks):
        dk = torch.zeros(ks[c].shape, device="cuda", dtype=torch.float32)
        dv = torch.zeros_like(dk)
        al = (bwd_alibi or {}).get(c, (slopes, dist0, ps))
        ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, scale, causal, off, 1, det, alibi=al)
        dks.append(dk)
        dvs.append(dv)
    return dict(o=out, lse=lse, dq=dq, dk=dks, dv=dvs)


def _oracle_chain(q, ks, vs, do, scale, chunks, slopes):
    masks = [("causal_offset", off) if causal else None for (causal, off), _ in chunks]
    return lm.oracle_chain(q, ks, vs, do, scale, masks, alibis=[(slopes, dist0, ps) for _, (dist0, ps) in chunks])


def _chain_errors(got, ref, dt):
    """Each output's relative error over its bound (O 2 u, gradients 4 u), and lse's over 2^-20 (1 + |lse|)."""
    cat = lambda d, k: torch.cat([t.detach().cpu().double() for t in d[k]], 1)  # noqa: E731
    r = {"o": _rel(got["o"], ref["o"]) / (2 * U[dt]), "dq": _rel(got["dq"], ref["dq"]) / (4 * U[dt]),
         "dk": _rel(cat(got, "dk"), cat(ref, "dk")) / (4 * U[dt]), "dv": _rel(cat(got, "dv"), cat(ref, "dv")) / (4 * U[dt])}
    g, l = got["lse"].detach().cpu().double(), ref["lse"]
    dead = torch.isinf(l) & (l < 0)
    r["lse_dead"] = 0.0 if torch.equal(torch.isinf(g) & (g < 0), dead) else float("inf")
    r["lse"] = float(((g - l).abs() / (1 + l.abs()))[~dead].max()) / 2.0 ** -20 if (~dead).any() else 0.0
    return r


# (name, Sq, [(Sk, (causal, off), (dist0, pstride))], slopes of the 2 heads)
CHAINS = [
    # a near chunk, then far ones: the carried lse is small, the later chunks' reference distances large
    ("near_then_far", 200, [(300, (False, 0), (0, 1)), (256, (False, 0), (3_000_000, 1)),
                            (129, (False, 0), (-3_000_017, 1))], (0.84, 0.5)),
    ("far_then_near", 200, [(256, (False, 0), (3_000_000, 1)), (300, (True, 100), (100, 1))], (0.84, 0.5)),
    # every chunk far, small slopes: lse stays moderate, so the backward can be checked at these positions
    ("far_chain_small_slopes", 129, [(200, (False, 0), (3_000_000, 1)), (130, (False, 0), (2_999_800, 1)),
                                     (64, (False, 0), (-2_999_990, 3))], (3e-5, 1.7e-5)),
    # the ring's striped stride; rows 0..63 of the first chunk see no key (causal offset -64) and revive later
    ("striped_dead_first", 129, [(128, (True, -64), (-64 * 4, 4)), (200, (True, 10), (40, 4))], (0.3, 0.11)),
    # a tile across d = 0 in a chain, then a neighbour
    ("diag_then_next", 255, [(255, (False, 0), (0, 1)), (257, (False, 0), (255, 1))], (0.25, 0.0625)),
]


def _chain_inputs(name, Sq, chunks, sl, D, dt, Hkv):
    seed = zlib.crc32(name.encode()) % 1000
    H = 2 if Hkv in (1, 2) else Hkv
    q, do = _rand((1, Sq, H, D), dt, seed), _rand((1, Sq, H, D), dt, seed + 1)
    ks = [_rand((1, sk, Hkv, D), dt, seed + 2 + 2 * i) for i, (sk, _, _) in enumerate(chunks)]
    vs = [_rand((1, sk, Hkv, D), dt, seed + 3 + 2 * i) for i, (sk, _, _) in enumerate(chunks)]
    slopes = torch.tensor([list(sl)], dtype=torch.float32)
    return q, ks, vs, do, slopes, [(m, a) for _, m, a in chunks]


@pytest.mark.parametrize("D,dt,Hkv", [(128, BF16, 2), (64, FP16, 1)])
@pytest.mark.parametrize("chain", CHAINS, ids=lambda c: c[0])
def test_chunk_chains_alibi(chain, D, dt, Hkv):
    name, Sq, chunks, sl = chain
    q, ks, vs, do, slopes, spec = _chain_inputs(name, Sq, chunks, sl, D, dt, Hkv)
    scale = D ** -0.5
    got = _native_chain(q, ks, vs, do, scale, spec, slopes.cuda())
    ref = _oracle_chain(q, ks, vs, do, scale, spec, slopes)
    err = _chain_errors(got, ref, dt)
    assert max(err.values()) <= 1.0, f"{name}: error / bound {err}"
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)
    if dead.any():  # rows no chunk lets see a key: O = 0 and dQ = 0 exactly
        rows = dead[0].all(0)
        assert (got["o"][:, rows.cuda()] == 0).all() and (got["dq"][:, rows.cuda()] == 0).all()
    again = _native_chain(q, ks, vs, do, scale, spec, slopes.cuda(), det=True)
    twice = _native_chain(q, ks, vs, do, scale, spec, slopes.cuda(), det=True)
    for k in ("dq", "dk", "dv"):  # deterministic mode: bitwise reproducible
        a, b = (x[k] if k == "dq" else torch.cat(x[k], 1) for x in (again, twice))
        assert torch.equal(a, b), k


def _faults(spec, slopes):
    """Realistic kernel faults as (name, side, {chunk: wrong alibi}): one kernel of one chunk gets them."""
    out = []
    for side in ("fwd", "bwd"):
        # chunk 0 holds each row's nearest keys in the chains below, so a wrong distance there carries weight
        (_, (dist0, ps)) = spec[0]
        out.append((f"dist0_plus1_{side}_chunk0", side, {0: (slopes, dist0 + 1, ps)}))
        # the K/V head's slope under GQA (2 query heads per K/V head: head 1 takes head 0's)
        out.append((f"kv_head_slope_{side}", side, {c: (slopes[:, :1].expand(1, 2).contiguous(), d, p)
                                                     for c, (_, (d, p)) in enumerate(spec)}))
    return out


@pytest.mark.parametrize("chain", [CHAINS[0], CHAINS[3], CHAINS[4]], ids=lambda c: c[0])
def test_kernel_faults_are_rejected(chain):
    """A distance one off, or the slope of the K/V head, given to the forward only or the backward only, moves some
    output past its bound; the same chain without the fault is within it."""
    name, Sq, chunks, sl = chain
    q, ks, vs, do, slopes, spec = _chain_inputs(name, Sq, chunks, sl, 128, BF16, 1)
    ref = _oracle_chain(q, ks, vs, do, 128 ** -0.5, spec, slopes)
    sl_cuda = slopes.cuda()
    for fault, side, wrong in _faults(spec, sl_cuda):
        if fault.startswith("dist0") and spec[0][0][0]:
            continue  # under causal a distance one off shifts every visible pair of a row alike (see above)
        kw = {"fwd_alibi": wrong} if side == "fwd" else {"bwd_alibi": wrong}
        err = _chain_errors(_native_chain(q, ks, vs, do, 128 ** -0.5, spec, sl_cuda, **kw), ref, BF16)
        assert max(err.values()) > 1.0, f"{name}: fault {fault} stays within every bound {err}"


# --------------------------------------------------------------------------- #
# the ring on one device
# --------------------------------------------------------------------------- #
def _ring_jobs(world):
    S = 128 if world == 8 else 192

    def j(mode, dt, D, Hkv, S_local, window=(-1, -1), per_batch=False, **kw):
        return rh.ring_job(world, mode, dt, D, Hkv, S_local, B=1, window=window, slopes="bh" if per_batch else "h",
                           **kw)

    jobs = [j("none", BF16, 128, 2, S),
            j("zigzag", BF16, 128, 2, S, per_batch=True),
            j("striped", FP16, 64, 4, S),
            j("striped", BF16, 128, 2, S, causal=False),
            j("none", FP16, 64, 1, S, (S // 2, S // 2)),
            j("zigzag", BF16, 128, 2, S, (S + 40, -1)),
            j("striped", BF16, 128, 2, S, (20, 9), causal=False)]
    if world == 4:
        jobs += [j(m, BF16, 128, 2, S, intra=2, dq_groups=True) for m in ("none", "zigzag", "striped")]
        jobs += [j("zigzag", BF16, 128, 2, 320, l2=128, det=True)]
        jobs += [j("none", BF16, 128, 2, S, seq_dim=2)]
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
def test_ring_alibi(runs, job):
    rh.check_ring_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))
