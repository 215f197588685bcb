"""ALiBi in the 16-bit model and comparator of ``tests/lowp_model.py``.

``lowp_alibi_forward`` / ``lowp_alibi_backward`` restate what ``fwd_alibi_kernel`` and ``bwd_alibi_kernel``
(csrc/fwd_sm90.cuh, csrc/bwd_sm90.cuh) compute for ``alibi = (slopes [B, H], dist0, pstride)``, rounding where the
kernels round (DESIGN 5.1b) and otherwise as ``lowp_model`` does:

* distances: row a and key c are ``d = pstride (a - c) + dist0`` apart, an exact int64; each row's reference ``dref``
  is its smallest |d| over the chunk's keys (``alibi_dref``), lowered under a live carried state of lse m0 (log2
  units) to the truncated fp32 ``cap = max(0, -m0) / slope2`` when that is smaller (``alibi_carried_ref``);
* forward: the fp32 log2 scores get ``fp32(-slope2 (|d| - dref))`` (slope2 = slope log2(e) in fp32); the carried
  state enters as ``m = fma(slope2, dref, m0)``; lse is ``(m + log2 l - slope2 dref) ln2``;
* backward, per tile of 64 rows x 128 keys from k0: on a tile where d has one sign s the loader's row statistic is
  ``fma(slope2, fp32(s (pstride (q - k0) + dist0)), fp32(lse log2(e)))`` and the exponent adds the per-key term
  ``s slope2 pstride (c - k0)``; on a tile across d = 0 it adds ``-slope2 |d|``.

Slopes are indexed by the query head, under GQA too.  The fp64 side is ``alibi_oracle``'s chunk functions, with
``lowp_model.error_scales`` over the pair bias of each chunk; lse is held to ``scores_absmax`` in the kernel's frame
(``|q| |k| scale + slope (|d| - dref)``), where a chunk millions of positions away adds only a few ulps.

``ALIBI_MUTANTS`` are realistic single faults of the ALiBi arithmetic for the comparator's own tests
(``tests/test_lowp_alibi.py``, ``tests/test_gpu_alibi_edges.py``); ``ALIBI_SWEEP`` is the edge sweep both run.
"""
from __future__ import annotations

import torch

import alibi_oracle as ao
import lowp_band
import lowp_model as lm

lowp_band.install()  # band masks (the lower edge every ALiBi driver call carries) in lowp_model's visibility

F32 = torch.float32
LOG2E_F = torch.tensor(lm.LOG2E, dtype=F32)
LN2_F = torch.tensor(lm.LN2, dtype=F32)
NEG_INF = float("-inf")
TILE_M, TILE_N = 64, 128  # both kernels classify tiles of 64 rows (from a multiple of 64) x 128 keys

# One realistic fault each.  "_fwd" / "_bwd": only that kernel has the fault.
ALIBI_MUTANTS = (
    "sign_dmin_fwd",         # forward: a tile with dmin in [-pstride, -1] is taken as d >= 0 throughout
    "sign_dmax_fwd",         # forward: a tile with dmax in [1, pstride] is taken as d <= 0 throughout
    "sign_dmin_bwd",         # backward (alibi_tile_sign): the same for dmin
    "sign_dmax_bwd",         # backward (alibi_tile_sign): the same for dmax
    "key_term_no_pstride",   # forward: the per-key term of a one-sign tile is s slope j, without pstride
    "bwd_gqa_first_head",    # backward consumer uses the slope of the group's first query head (the loader does not)
    "carried_not_lowered",   # forward: the carried state's reference is not lowered (alibi_carried_ref skipped)
    "dist0_plus1_fwd",       # forward uses dist0 + 1
    "dist0_plus1_bwd",       # backward uses dist0 + 1
)


def _fma(a, b, c):
    """fp32 fma(a, b, c) of fp32 operands: the exact product in fp64, one rounding of the sum."""
    return (a.double() * b.double() + c.double()).to(F32)


def slope2_of(slopes):
    """[B, H] fp32: the slope in log2 units as the kernels load it."""
    return slopes.to(F32) * LOG2E_F.to(slopes.device)


def distances(sq, sk, dist0, pstride, device=None):
    """int64 [sq, sk]: d = pstride (a - c) + dist0."""
    a = torch.arange(sq, dtype=torch.int64, device=device).view(-1, 1)
    c = torch.arange(sk, dtype=torch.int64, device=device).view(1, -1)
    return pstride * (a - c) + int(dist0)


def alibi_dref(sq, sk, dist0, pstride, device=None):
    """int64 [sq]: each row's smallest |d| over keys 0 .. sk-1 (0 when d changes sign)."""
    hi = pstride * torch.arange(sq, dtype=torch.int64, device=device) + int(dist0)  # d at key 0
    lo = hi - pstride * (sk - 1)                                                    # d at key sk-1
    return torch.maximum(lo, -hi).clamp(min=0)


def dref_source(sq, sk, dist0, pstride):
    """[sq] str per row: "key0" (d < 0 throughout), "keylast" (d > 0 throughout) or "zero" (dref = 0)."""
    hi = pstride * torch.arange(sq, dtype=torch.int64) + int(dist0)
    lo = hi - pstride * (sk - 1)
    return ["key0" if h < 0 else "keylast" if l > 0 else "zero" for h, l in zip(hi.tolist(), lo.tolist())]


def carried_ref(dref, m0, slope2):
    """``alibi_carried_ref``: dref [B,H,Sq] int64 lowered to trunc(max(0, -m0) / slope2) where that (fp32) is
    smaller; m0 fp32 [B,H,Sq] (log2 units), slope2 fp32 [B,H].  Returns (dref, lowered mask)."""
    s2 = slope2.unsqueeze(-1)
    cap = torch.clamp(-m0, min=0.0) / torch.where(s2 > 0, s2, torch.ones_like(s2))
    low = (s2 > 0) & (cap < dref.to(F32)) & torch.isfinite(cap)
    return torch.where(low, cap.to(torch.int64), dref), low


def tile_bounds(sq, sk, dist0, pstride, device=None):
    """int64 [sq, sk]: (dmin, dmax) of the 64 x 128 tile each pair lies in, over the tile's whole geometry."""
    R = (torch.arange(sq, dtype=torch.int64, device=device) // TILE_M * TILE_M).view(-1, 1)
    K = (torch.arange(sk, dtype=torch.int64, device=device) // TILE_N * TILE_N).view(1, -1)
    dmin = pstride * (R - K - (TILE_N - 1)) + int(dist0)
    dmax = pstride * (R + TILE_M - 1 - K) + int(dist0)
    return dmin, dmax


def tile_sign(sq, sk, dist0, pstride, device=None, mutant=None, side="fwd"):
    """int64 [sq, sk]: the sign the kernel gives each pair's tile, +1 / -1 (one sign, 0 counted with either) or 0
    (across d = 0); the "sign_*" mutants misclassify the tiles one sign edge away."""
    dmin, dmax = tile_bounds(sq, sk, dist0, pstride, device)
    s = torch.where(dmin >= 0, 1, torch.where(dmax <= 0, -1, 0))
    if mutant == "sign_dmin_" + side:
        s = torch.where((dmin >= -pstride) & (dmin <= -1), 1, s)
    if mutant == "sign_dmax_" + side:
        s = torch.where((dmax >= 1) & (dmax <= pstride), -1, s)
    return s


def _alibi_of(alibi, side, mutant):
    slopes, dist0, ps = alibi
    return slopes, int(dist0) + (1 if mutant == "dist0_plus1_" + side else 0), int(ps)


def lowp_alibi_forward(q, k, v, scale, mask, alibi, state=None, last=True, mutant=None, info=None):
    """One forward chunk with carried state, rounded like ``fwd_alibi_kernel``.  Arguments and result as
    ``lowp_model.lowp_forward``; ``alibi = (slopes fp32 [B, H], dist0, pstride)``; ``info`` (a dict), if given,
    counts the live carried rows whose reference was lowered ("lowered") and those with dref > 0 it left alone
    ("kept")."""
    dtype = q.dtype
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    dev = q.device
    slopes, dist0, ps = _alibi_of(alibi, "fwd", mutant)
    slope2 = slope2_of(slopes.to(dev))  # [B,H]
    kk, vv = lm._kv_heads(k, H), lm._kv_heads(v, H)
    d = distances(Sq, Sk, dist0, ps, dev)
    sg = tile_sign(Sq, Sk, dist0, ps, dev, mutant, "fwd")
    ad = torch.where(sg == 0, d.abs(), sg * d)  # |d| as the tile forms it
    if mutant == "key_term_no_pstride":
        j = torch.arange(Sk, dtype=torch.int64, device=dev).view(1, -1) % TILE_N
        ad = torch.where(sg == 0, ad, ad + sg * (ps - 1) * j)
    dref = alibi_dref(Sq, Sk, dist0, ps, dev).view(1, 1, Sq).expand(B, H, Sq)
    m0 = None
    if state is not None:
        o0 = state[0].float().permute(0, 2, 1, 3)  # [B,H,Sq,D]
        lse0 = state[1].float()
        alive = lse0 != NEG_INF
        m0 = lse0 * LOG2E_F.to(dev)
        if mutant != "carried_not_lowered":
            low_ref, low = carried_ref(dref, torch.where(alive, m0, torch.zeros_like(m0)), slope2)
            dref = torch.where(alive, low_ref, dref)
            if info is not None:
                info["lowered"] = info.get("lowered", 0) + int((low & alive).sum())
                info["kept"] = info.get("kept", 0) + int((~low & alive & (dref > 0)).sum())
    dref_f = dref.to(F32)
    x = (ad.view(1, 1, Sq, Sk) - dref.unsqueeze(-1)).to(F32)  # |d| - dref, exact integer (fp32 above 2^24)
    bias2 = (-slope2.double().view(B, H, 1, 1) * x.double()).to(F32)
    raw = torch.einsum("bqhd,bkhd->bhqk", q.float(), kk.float())
    s = raw * lm._scale_log2(scale) + bias2
    vis = lowp_band.visible(Sq, Sk, mask, dev)
    if vis is not None:
        s = s.masked_fill(~vis, NEG_INF)
    m = s.amax(-1)
    if state is not None:
        m_c = _fma(slope2.view(B, H, 1).expand(B, H, Sq), dref_f, m0)  # m0 + slope2 dref: the row's frame
        m = torch.where(alive, torch.maximum(m, m_c), m)
    msafe = torch.where(m == NEG_INF, torch.zeros_like(m), m)
    p = torch.exp2(s - msafe.unsqueeze(-1))
    l = p.sum(-1)
    o = torch.einsum("bhqk,bhkd->bhqd", lm._round(p, dtype), vv.float().permute(0, 2, 1, 3))
    if state is not None:
        f = torch.where(alive, torch.exp2(m_c - msafe), torch.zeros_like(m))
        l = l + alive.float() * f
        o = o + o0 * f.unsqueeze(-1)
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    o = (o * inv.unsqueeze(-1)).permute(0, 2, 1, 3).contiguous()
    t = m + torch.log2(torch.where(l > 0, l, torch.ones_like(l)))
    lse = torch.where(l > 0, _fma(-slope2.view(B, H, 1).expand(B, H, Sq), dref_f, t) * LN2_F.to(dev),
                      torch.full_like(l, NEG_INF))
    return (o.to(dtype) if last else o), lse


def lowp_alibi_backward(q, k, v, do, o, lse, scale, mask, alibi, mutant=None):
    """One backward chunk, rounded like ``delta_kernel`` + ``bwd_alibi_kernel``; as ``lowp_model.lowp_backward``."""
    dtype = q.dtype
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    dev = q.device
    slopes, dist0, ps = _alibi_of(alibi, "bwd", mutant)
    slope2 = slope2_of(slopes.to(dev))  # [B,H]
    slope_key = slope2
    if mutant == "bwd_gqa_first_head":
        G = H // Hkv
        slope_key = slope2[:, torch.arange(H, device=dev) // G * G]
    kk, vv = lm._kv_heads(k, H), lm._kv_heads(v, H)
    delta = (o.float() * do.float()).sum(-1).permute(0, 2, 1)  # [B,H,Sq]
    d = distances(Sq, Sk, dist0, ps, dev)
    sg = tile_sign(Sq, Sk, dist0, ps, dev, mutant, "bwd")
    a = torch.arange(Sq, dtype=torch.int64, device=dev).view(-1, 1)
    c = torch.arange(Sk, dtype=torch.int64, device=dev).view(1, -1)
    k0 = c // TILE_N * TILE_N
    row_term = sg * (ps * (a - k0) + dist0)                               # 0 across d = 0
    key_term = torch.where(sg == 0, -d.abs(), sg * ps * (c - k0))
    lse2 = torch.where(lse == NEG_INF, torch.full_like(lse, float("inf")), lse.float()) * LOG2E_F.to(dev)
    stat = _fma(slope2.view(B, H, 1, 1), row_term.to(F32).view(1, 1, Sq, Sk), lse2.unsqueeze(-1))
    x0 = _fma(slope_key.view(B, H, 1, 1), key_term.to(F32).view(1, 1, Sq, Sk), -stat)
    raw = torch.einsum("bqhd,bkhd->bhqk", q.float(), kk.float())
    p = torch.exp2(_fma(raw, torch.tensor(lm._scale_log2(scale), dtype=F32), x0))
    vis = lowp_band.visible(Sq, Sk, mask, dev)
    if vis is not None:
        p = p.masked_fill(~vis, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", lm._round(p, dtype), do.float())
    dp = torch.einsum("bqhd,bkhd->bhqk", do.float(), vv.float())
    ds = lm._round(p * (dp - delta.unsqueeze(-1)), dtype)
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk.float()) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q.float()) * scale
    return dq, lm._group_sum(dk, Hkv), lm._group_sum(dv, Hkv)


# --------------------------------------------------------------------------- #
# chains: the model and the fp64 oracle side by side
# --------------------------------------------------------------------------- #
def lowp_alibi_chain(q, ks, vs, do, scale, masks, alibis, mutant=None, lse_bwd=None, info=None):
    """``lowp_model.lowp_chain`` with ALiBi (``alibis[c] = (slopes, dist0, pstride)`` of chunk c).

    ``lse_bwd``: the fp32 lse the backward reads (default: the model's own).  A kernel test passes the kernels' own:
    far from d = 0 the backward turns the fp32 rounding of lse itself (ulp(slope dref), DESIGN 5.1b) into an error of
    P that the model reproduces only from the same lse; the lse is held to the oracle on its own."""
    n = len(ks)
    state, states = None, []
    for c in range(n):
        o, lse = lowp_alibi_forward(q, ks[c], vs[c], scale, masks[c], alibis[c], state, last=c == n - 1,
                                    mutant=mutant, info=info)
        if c < n - 1:
            state = (o, lse)
            states.append(state)
    lb = lse if lse_bwd is None else lse_bwd.to(q.device)
    dq = torch.zeros(q.shape, device=q.device, dtype=torch.float32)
    dks, dvs = [], []
    for c in range(n):
        dqc, dk, dv = lowp_alibi_backward(q, ks[c], vs[c], do, o, lb, scale, masks[c], alibis[c], mutant=mutant)
        dq += dqc
        dks.append(dk)
        dvs.append(dv)
    return dict(o=o, lse=lse, states=states, dq=dq, dk=dks, dv=dvs)


def oracle_alibi_chain(q, ks, vs, do, scale, masks, alibis):
    """The same chain in fp64 (``alibi_oracle``, CPU), with ``lowp_model.error_scales`` over each chunk's bias."""
    n = len(ks)
    cpu = lambda t: t.detach().cpu()  # noqa: E731
    q, do = cpu(q), cpu(do)
    H, Hkv = q.shape[2], ks[0].shape[2]
    kx = [lm._kv_heads(cpu(k), H) for k in ks]
    vx = [lm._kv_heads(cpu(v), H) for v in vs]
    al = [(cpu(s), d0, ps) for s, d0, ps in alibis]
    o, lse, states = None, None, []
    for c in range(n):
        o, lse = ao.chunk_forward(q, kx[c], vx[c], o, lse, scale, masks[c], al[c])
        if c < n - 1:
            states.append((o, lse))
    delta = (o * do.double()).sum(-1).permute(0, 2, 1)
    lse_b = torch.where(torch.isinf(lse), torch.full_like(lse, float("inf")), lse)  # dead rows: P = 0
    dq = torch.zeros(q.shape, dtype=torch.float64)
    dks, dvs = [], []
    for c in range(n):
        dqc, dk, dv = ao.chunk_backward(do, q, kx[c], vx[c], delta, lse_b, scale, masks[c], al[c])
        dq += dqc
        dks.append(lm._group_sum(dk, Hkv))
        dvs.append(lm._group_sum(dv, Hkv))
    biases = [ao.chunk_bias(al[c], q.shape[1], kx[c].shape[1]) for c in range(n)]
    return dict(o=o, lse=lse, states=states, dq=dq, dk=dks, dv=dvs,
                **lm.error_scales(q, kx, vx, do, o, delta, lse_b, scale, masks, biases, Hkv))


def frame_bias(alibi, sq, sk):
    """fp64 [B,H,Sq,Sk]: the bias in the kernel's frame, -slope (|d| - dref) (the chunk's own dref)."""
    slopes, dist0, ps = alibi
    x = distances(sq, sk, dist0, ps).abs() - alibi_dref(sq, sk, dist0, ps).view(-1, 1)
    return -slopes.detach().cpu().double().view(*slopes.shape, 1, 1) * x.double()


def absmax_prefix(q, ks, scale, masks, alibis):
    """``lowp_model.scores_absmax`` over chunks 0..c for every c, in the kernel's frame."""
    sq = q.shape[1]
    fb = [frame_bias(a, sq, k.shape[1]) for a, k in zip(alibis, ks)]
    return [lm.scores_absmax(q, ks[:c + 1], scale, masks[:c + 1], fb[:c + 1]) for c in range(len(ks))]


# --------------------------------------------------------------------------- #
# the ALiBi edge sweep (tests/test_gpu_alibi_edges.py on the kernels, tests/test_lowp_alibi.py on the model)
# --------------------------------------------------------------------------- #
# A case: Sq rows against a chain of chunks (Sk, mask, dist0) with one pstride, slopes of a kind, and the
# lowp_model case fields (head dim, dtype, batch / heads, layout) that seed and shape the inputs.
BF16, FP16 = torch.bfloat16, torch.float16
FAR = 3_000_000


def slopes_for(kind, B, H):
    """fp32 [B, H] slopes of a kind: "std" (flash-attn's), "large" (0.5 .. 1), "tiny" (1e-5), "zero", "neg" (the
    standard ones with the first head's at -0.25) or "bh" (per (batch, head))."""
    std = ao.std_slopes(H).view(1, H).expand(B, H)
    if kind == "std":
        return std.contiguous()
    if kind == "large":
        return torch.linspace(0.5, 1.0, H).view(1, H).expand(B, H).contiguous()
    if kind == "tiny":
        return torch.full((B, H), 1e-5)
    if kind == "zero":
        return torch.zeros(B, H)
    if kind == "neg":
        s = std.clone()
        s[:, 0] = -0.25
        return s
    assert kind == "bh", kind
    return ao.slopes_for(B, H, True, seed=5)


def _mask_id(m):
    if m is None:
        return ""
    if m[0] == "causal_offset":
        return f"c{m[1]}"
    return f"b{m[1]}_{m[2]}"


def acase(sq, chunks, ps=1, slopes="std", D=128, dtype=BF16, B=1, H=2, Hkv=None, layout="flash", tag=""):
    """chunks: [(Sk, mask, dist0)] with mask None, ("causal_offset", off) or ("band", lo, hi)."""
    ch = "+".join(f"{_mask_id(m)}d{d0}" for _, m, d0 in chunks) if len(chunks) <= 3 else f"d{chunks[0][2]}"
    c = lm._case(sq, [(sk, None) for sk, _, _ in chunks], D, dtype, B=B, H=H, Hkv=Hkv, layout=layout,
                 tag=f"alibi_{tag}p{ps}_{slopes}_{ch}_")
    c.update(masks=[m for _, m, _ in chunks], dist0s=[d0 for _, _, d0 in chunks], ps=ps, slopes=slopes)
    return c


def view_chain(sizes, dist0, ps, causal=False):
    """Chunks of one problem: keys of chunk c start sum(sizes[:c]) keys later, so dist0 drops by ps per key; causal:
    the causal mask where d >= 0 (dist0 a multiple of ps)."""
    out, k0 = [], 0
    for sk in sizes:
        d0 = dist0 - ps * k0
        out.append((sk, ("causal_offset", d0 // ps) if causal else None, d0))
        k0 += sk
    return out


def _sweep():
    cs = []
    dts = [(128, BF16), (64, FP16), (64, BF16), (128, FP16)]
    # sign edges: per pstride, a chain whose chunks put tile (0, 0)'s dmin on 0, -1 and -pstride, and one whose chunks
    # put its dmax on 0, 1 and pstride (a chunk is any view: its dist0 is its own)
    shapes = [(129, 257, 128, 383), (65, 513, 255, 1), (255, 127, 63, 129), (383, 64, 513, 257), (63, 129, 257, 65)]
    for i, ps in enumerate((1, 2, 3, 4, 8)):
        sq, a, b, c = shapes[i]
        D, dt = dts[i % 4]
        lo = [127 * ps, 127 * ps - 1, 126 * ps]   # dmin 0, -1, -ps
        hi = [-63 * ps, -63 * ps + 1, -62 * ps]   # dmax 0, 1, ps
        cs.append(acase(sq, [(a, None, lo[0]), (b, None, lo[1]), (c, None, lo[2])], ps, "large", D, dt, tag="dmin_"))
        D, dt = dts[(i + 1) % 4]
        cs.append(acase(sq, [(b, None, hi[0]), (c, None, hi[1]), (a, None, hi[2])], ps, "large" if i < 3 else "std",
                        D, dt, tag="dmax_"))
    # the same edges one tile row / column further on, and at +-64 ps and +-128 ps, +-1 and +-ps, one chunk each
    for i, (ps, d0) in enumerate([(1, 64), (1, -64), (1, 128 + 1), (1, -128 - 1), (2, 2 * 64 + 2), (2, -2 * 128 - 2),
                                  (3, 3 * 128 - 1), (3, -3 * 64 + 3), (4, 4 * 127 + 4 * 64), (8, -8 * 63 - 8 * 64 + 8),
                                  (8, 8 * 127 - 8 * 64 - 1), (4, -4 * 63 + 4 * 128 + 1)]):
        D, dt = dts[i % 4]
        sq, sk = [(257, 513), (383, 255), (129, 383), (513, 129), (255, 257), (65, 513)][i % 6]
        cs.append(acase(sq, [(sk, None, d0)], ps, ["std", "large"][i % 2], D, dt))
    # d never 0: pstride does not divide dist0, across and beside d = 0
    cs.append(acase(257, [(257, None, 5), (129, None, 3 * 127 + 1)], 3, "large", 128, BF16, tag="nozero_"))
    cs.append(acase(129, [(383, None, -8 * 63 - 3)], 8, "std", 64, FP16, tag="nozero_"))
    # one row / one key
    cs.append(acase(1, [(513, None, 200)], 1, "large", 128, FP16))
    cs.append(acase(383, [(1, None, -127)], 2, "std", 64, BF16))
    # causal masks on the edges: views of one causal problem (d >= 0 visible), and offsets that do not meet d = 0
    for i, ps in enumerate((1, 2, 4)):
        D, dt = dts[i % 4]
        cs.append(acase(257, [(383, ("causal_offset", 127), 127 * ps)], ps, "large", D, dt, tag="causal_"))
        cs.append(acase(129, view_chain([128, 129], 128 * ps, ps, causal=True), ps, "std", D, dt, tag="causal_"))
    cs.append(acase(255, [(257, ("causal_offset", 1), 64)], 1, "large", 128, FP16, tag="causal_"))
    cs.append(acase(129, [(513, ("causal_offset", -64), -63)], 1, "std", 64, BF16, tag="causal_"))
    # band lower edge with ALiBi (every driver call runs the band launches)
    cs.append(acase(257, [(257, ("band", -100, 0), 0)], 1, "large", 128, BF16, tag="band_"))
    cs.append(acase(200, [(383, ("band", -64, 63), 127)], 2, "std", 64, FP16, tag="band_"))
    cs.append(acase(129, [(257, ("band", 150, None), 0)], 1, "std", 128, FP16, tag="band_"))  # rows from 107 dead
    # distance: near->far, far->near, far->far and 16-chunk chains, views of one problem, at large slopes
    for D, dt in [(128, BF16), (64, FP16)]:
        cs.append(acase(129, [(257, None, 100), (128, None, FAR)], 1, "large", D, dt, tag="nearfar_"))
        cs.append(acase(129, [(257, None, FAR), (200, None, 60)], 1, "large", D, dt, tag="farnear_"))
        cs.append(acase(255, view_chain([128, 129], FAR, 1), 1, "large", D, dt, tag="farfar_"))
        cs.append(acase(129, view_chain([64] * 16, -FAR + 1024, 2), 2, "large", D, dt, tag="farfar_"))
        cs.append(acase(129, view_chain([64] * 16, 600, 1), 1, "std", D, dt, tag="chain16_"))
    cs.append(acase(129, [(257, None, -40), (255, None, -FAR - 7)], 3, "large", 128, BF16, tag="nearfar_"))
    cs.append(acase(65, view_chain([128, 64, 129], 2 ** 24 + 3, 1), 1, "large", 128, BF16, tag="2p24_"))
    cs.append(acase(129, [(257, None, -(2 ** 24) - 5)], 1, "std", 64, FP16, tag="2p24_"))
    # slopes: tiny, zero, negative, per (batch, head)
    cs.append(acase(129, [(257, None, 100), (128, None, FAR)], 1, "tiny", 128, BF16))
    cs.append(acase(257, [(255, None, 0)], 1, "tiny", 64, FP16))
    cs.append(acase(129, [(257, None, 60), (129, None, -200)], 1, "zero", 128, FP16))
    cs.append(acase(255, [(257, None, 40), (129, None, 1000)], 1, "neg", 128, BF16))
    cs.append(acase(129, [(383, ("causal_offset", 254), 254)], 1, "neg", 64, FP16))
    cs.append(acase(129, [(257, None, 127), (128, None, FAR)], 2, "bh", 128, BF16, B=2))
    cs.append(acase(255, [(129, None, -63)], 1, "bh", 64, FP16, B=2))
    # grouped-query attention, a distinct slope per query head
    for i, hkv in enumerate((4, 2, 1)):
        D, dt = dts[i % 4]
        cs.append(acase(129, [(257, None, 127 - 64 * i)], 1, "large", D, dt, H=8, Hkv=hkv))
    cs.append(acase(255, [(257, ("causal_offset", 0), 0)], 4, "std", 128, FP16, H=4, Hkv=1))
    # layouts
    for D, dt in [(128, FP16), (64, BF16)]:
        cs.append(acase(129, [(257, ("causal_offset", 127), 127)], 1, "std", D, dt, B=2, layout="bstride"))
        cs.append(acase(255, [(129, None, -64), (128, None, FAR)], 2, "large", D, dt, layout="normal"))
        cs.append(acase(129, [(257, None, 0)], 1, "bh", D, dt, B=2, H=4, Hkv=2, layout="bstride"))
    ids = [c["id"] for c in cs]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    return cs


ALIBI_SWEEP = _sweep()


def _pick(tag, dtype, ps=None, H=None):
    """The id of the first sweep case with this tag (after "alibi_"), dtype, pstride and head count."""
    for c in ALIBI_SWEEP:
        if c["id"].startswith("alibi_" + tag) and c["dtype"] == dtype and (ps is None or c["ps"] == ps) and \
                (H is None or c["H"] == H):
            return c["id"]
    raise LookupError((tag, dtype, ps, H))


# per mutant: one bf16 and one fp16 case of the sweep on which the fault is live
MUTANT_CASES = {
    "sign_dmin_fwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "sign_dmax_fwd": [_pick("dmax_", BF16, 2), _pick("dmax_", FP16, 1)],
    "sign_dmin_bwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "sign_dmax_bwd": [_pick("dmax_", BF16, 2), _pick("dmax_", FP16, 1)],
    "key_term_no_pstride": [_pick("dmin_", BF16, 3), _pick("dmin_", FP16, 2)],
    "bwd_gqa_first_head": [_pick("p1_large", BF16, 1, H=8), _pick("p1_large", FP16, 1, H=8)],
    "carried_not_lowered": [_pick("nearfar_", BF16, 1), _pick("nearfar_", FP16, 1)],
    "dist0_plus1_fwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "dist0_plus1_bwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
}


def make_alibi_inputs(case, device="cpu"):
    """``lowp_model.make_inputs`` of the case plus its masks and ``alibis[c] = (slopes fp32 [B, H], dist0,
    pstride)`` on ``device``."""
    x = lm.make_inputs(case, device)
    x["masks"] = list(case["masks"])
    slopes = slopes_for(case["slopes"], case["B"], case["H"]).to(device)
    x["alibis"] = [(slopes, d0, case["ps"]) for d0 in case["dist0s"]]
    return x


def tile_classes(case):
    """The sign classes the case's tiles hit (both kernels classify 64 x 128 tiles), as a set of tuples:
    ("dmin", value, ps) for dmin in {0, -1, -ps}, ("dmax", value, ps) for dmax in {0, 1, ps}, ("cross", ps),
    ("nozero", ps) for a crossing tile where ps does not divide dist0, and ("dref", source) per row."""
    out = set()
    ps = case["ps"]
    sk_of = [sk for sk, _ in case["chunks"]]
    for sk, d0 in zip(sk_of, case["dist0s"]):
        for R in range(0, case["sq"], TILE_M):
            for K in range(0, sk, TILE_N):
                dmin = ps * (R - K - (TILE_N - 1)) + d0
                dmax = ps * (R + TILE_M - 1 - K) + d0
                if dmin in (0, -1, -ps):
                    out.add(("dmin", dmin, ps))
                if dmax in (0, 1, ps):
                    out.add(("dmax", dmax, ps))
                if dmin < 0 < dmax:
                    out.add(("cross", ps))
                    if d0 % ps:
                        out.add(("nozero", ps))
        out.update(("dref", s) for s in dref_source(case["sq"], sk, d0, ps))
    return out
