"""A 16-bit rounding model of the tile kernels, and the comparator the tile-edge tests use.

``lowp_forward`` / ``lowp_backward`` restate what ``fwd_chunk_kernel`` (csrc/fwd_sm90.cu) and ``bwd_chunk_kernel``
(csrc/bwd_sm90.cu) compute, rounding at the same points the kernels round and nowhere else:

* scores are fp32 products of the 16-bit inputs, taken to log2 units with the fp32 ``scale * log2(e)``; a key bias
  is added in log2 units;
* forward: the softmax runs in fp32; its row sum ``l`` adds the unrounded P; P is rounded to the input dtype
  (``pack2``) before ``P V``, which accumulates in fp32; the carried state enters as ``m = lse log2(e)``, ``l = 1``,
  ``acc = o_acc`` (fp32, normalised); O is rounded once, at the end of the last chunk;
* backward: delta = rowsum(O dO) in fp32 from the 16-bit O; P is recomputed in fp32 from the final lse; ``dV`` uses P
  rounded to 16 bit; ``dS = P (dP - delta)`` is rounded to 16 bit before both ``dQ = dS K`` and ``dK = dS^T Q``, which
  accumulate in fp32 and are multiplied by the (fp32) scale.

The model does not reproduce the kernels' order of fp32 operations (the kernel rounds P relative to the running
maximum of its key tile, the model relative to the final row maximum), so it is a yardstick of the same error
magnitude, not a bitwise twin.  The truth is ``mask_oracle`` (``oracle/attention_oracle.py`` for the masks it states)
in fp64 on the same 16-bit inputs.

Masks are the kernels' (``mask_oracle.mask_of``): ``None``, ``("causal_offset", off)`` (key b visible to row a iff
``b <= a + off``), the band ``("band", lo, hi)`` and the document mask ``("doc", lo, hi, cu, q_pos0, k_pos0, pstride)``.
A chunk may also carry ALiBi, ``(slopes [B, H], dist0, pstride)``: ``lowp_alibi_forward`` / ``lowp_alibi_backward``
restate the ALiBi kernels' own arithmetic, which differs from the plain kernels' (below).  Tensors are in the flash
layout ``[B, S, H, D]``; K/V may have fewer heads than Q (query head h reads K/V head ``h // G``).  The model runs on
whatever device its inputs live on.

``mutant`` injects one realistic kernel fault into the model: ``MUTANTS`` here, ``lowp_band.BAND_MUTANTS`` at the
band's lower edge, ``lowp_doc.DOC_MUTANTS`` in the document kernels' index arithmetic (restated in ``doc_index``) and
``lowp_alibi.ALIBI_MUTANTS`` in the ALiBi arithmetic.  ``tests/test_lowp_{model,band,doc,alibi}.py`` show that the
comparator rejects each of them.
"""
from __future__ import annotations

import torch

import doc_index as di
import mask_oracle as mo
from oracle import attention_oracle as orc

LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
NEG_INF = float("-inf")

# One realistic fault each, for the comparator's own tests.  "_fwd" / "_bwd": only that kernel has the fault.
MUTANTS = (
    "drop_key_127",         # key 127 never contributes (forward and backward)
    "drop_key_128",         # key 128 never contributes
    "drop_key_last",        # the last key (the ragged tail) never contributes
    "causal_plus1_fwd",     # forward causal limit one key too large
    "causal_minus1_fwd",    # forward causal limit one key too small
    "causal_plus1_bwd",     # backward causal mask lets one key too many through
    "causal_minus1_bwd",    # backward causal mask drops the diagonal key
    "strict_swap",          # b < a + off where b <= a + off belongs (both kernels)
    "scale_fwd",            # forward uses scale * (1 + 2^-8)
    "scale_bwd",            # backward uses scale * (1 + 2^-8)
    "bias_natural_fwd",     # forward adds the key bias in natural units to log2-unit scores
    "bias_natural_bwd",     # backward does the same
    "carried_l4",           # carried state loaded with l = 4 instead of 1 (lse counted twice over)
    "dead_revive_stale_m",  # a row dead in the carried state is loaded as if its lse were 0
    "gqa_wrong_head",       # the last query head reads K/V head (h // G + 1) mod Hkv
    "dk_no_scale",          # dK not multiplied by scale
    "dq_missing_key_block", # dQ misses the partial of one 128-key block
    "dv_missing_q_block",   # dV misses the first 64-row Q block a causal key block sees (i_begin one block late)
)


def unit_roundoff(dtype: torch.dtype) -> float:
    return {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dtype]


def _round(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    return x.to(dtype).to(torch.float32)


def _scale_log2(scale: float) -> float:
    return float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))


def visible(sq: int, sk: int, mask, device=None, shift: int = 0, strict: bool = False, lo_shift: int = 0):
    """[sq, sk] bool visibility of ``mask`` (None: everything visible).  Mutant hooks: ``shift`` / ``strict`` act on
    the causal offset or the band's upper edge, ``lo_shift`` moves the band's lower edge that many keys down."""
    if mask is None:
        return None
    a = torch.arange(sq, device=device).unsqueeze(1)
    b = torch.arange(sk, device=device).unsqueeze(0)
    if mask[0] == "causal_offset":
        off = int(mask[1])
        return b < a + off + shift if strict else b <= a + off + shift
    assert mask[0] in ("band", "doc"), mask
    lo, hi = mask[1], mask[2]
    m = torch.ones(sq, sk, dtype=torch.bool, device=device)
    if lo is not None:
        m &= b >= a + int(lo) - lo_shift
    if hi is not None:
        m &= (b < a + int(hi) + shift) if strict else (b <= a + int(hi) + shift)
    if mask[0] == "doc":
        _, _, _, cu, q_pos0, k_pos0, ps = mask
        m &= mo.same_doc(q_pos0 + ps * torch.arange(sq), k_pos0 + ps * torch.arange(sk), list(cu)).to(device)
    return m


def _kv_heads(t: torch.Tensor, H: int, mutant=None) -> torch.Tensor:
    """K or V [B, Sk, Hkv, D] -> [B, Sk, H, D]: query head h reads K/V head h // G."""
    Hkv = t.shape[2]
    G = H // Hkv
    idx = torch.arange(H, device=t.device) // G
    if mutant == "gqa_wrong_head":
        idx[H - 1] = (idx[H - 1] + 1) % Hkv
    return t.index_select(2, idx)


def _group_sum(t: torch.Tensor, Hkv: int) -> torch.Tensor:
    B, S, H, D = t.shape
    return t.view(B, S, Hkv, H // Hkv, D).sum(3)


def _drop_keys(sk: int, mutant) -> list:
    return {"drop_key_127": [127], "drop_key_128": [128], "drop_key_last": [sk - 1]}.get(mutant, [])


def _scores_log2(q, k, scale, key_bias, mutant, side):
    """fp32 scores in log2 units [B, H, Sq, Sk] (+ the key bias in log2 units)."""
    if mutant == "scale_" + side:
        scale = scale * (1 + 2.0 ** -8)
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * _scale_log2(scale)
    if key_bias is not None:
        b = key_bias.float() * (1.0 if mutant == "bias_natural_" + side else LOG2E)
        s = s + b.unsqueeze(2)
    return s


def _vis_for(sq, sk, mask, device, mutant, side):
    """``visible`` as the ``side`` ("fwd" / "bwd") kernel computes it with the fault ``mutant``."""
    if mask is not None and mask[0] == "band":
        return _band_vis_for(sq, sk, mask, device, mutant, side)
    if mask is not None and mask[0] == "doc":
        return _doc_vis_for(sq, sk, mask, device, mutant, side)
    shift = {"causal_plus1_" + side: 1, "causal_minus1_" + side: -1}.get(mutant, 0)
    return visible(sq, sk, mask, device, shift=shift, strict=mutant == "strict_swap")


# --------------------------------------------------------------------------- #
# the band kernels' index arithmetic (fwd_sm90.cuh, bwd_sm90.cuh) for one band launch, and the band's faults
# --------------------------------------------------------------------------- #
TILE_F, TILE_N, TILE_M = 128, 128, 64  # forward: 128 rows x 128 keys (two 64-row warpgroups); backward: 128 x 64


def fwd_trip_count(r0, sq, sk, hi):
    """One past the last 128-key tile the 64 rows from r0 visit (``fwd_trip_count``); hi None: not causal."""
    if r0 >= sq:
        return 0
    lim = sk - 1 if hi is None else min(min(r0 + 63, sq - 1) + hi, sk - 1)
    return 0 if lim < 0 else lim // TILE_N + 1


def fwd_first_tile(r0, lo):
    """The first tile the 64 rows from r0 visit (``fwd_first_tile``)."""
    return max(0, r0 + lo) // TILE_N


def bwd_q_range(k0, sq, sk, lo, hi):
    """(i_begin, i_end): the 64-row Q blocks key block k0 visits (``bwd_chunk_body``)."""
    nq = (sq + TILE_M - 1) // TILE_M
    ib = 0 if hi is None else max(0, k0 - hi) // TILE_M
    ql = min(k0 + TILE_N - 1, sk - 1) - lo
    ie = 0 if ql < 0 else min(nq, ql // TILE_M + 1)
    return ib, ie


def host_lower(sq, sk, lo, mutant=None):
    """The lower edge the kernels get from ``check_chunk_args`` (csrc/host_common.cu) (None: dropped, the kernel without one runs)."""
    if lo is None:
        return None
    if lo <= (2 if mutant == "band_drop_at_2_minus_sq" else 1) - sq:
        return None
    if lo > sk:
        return sk - 1 if mutant == "band_clamp_sk_minus1" else sk
    return lo


def _band_vis_for(sq, sk, mask, device, mutant, side):
    """``_vis_for`` of a band: the causal mutants act on its upper edge, ``lowp_band.BAND_MUTANTS`` on its lower."""
    _, lo, hi = mask
    if mutant in ("band_drop_at_2_minus_sq", "band_clamp_sk_minus1"):
        lo = host_lower(sq, sk, lo, mutant)
    mask = ("band", lo, hi)
    shift = {"causal_plus1_" + side: 1, "causal_minus1_" + side: -1}.get(mutant, 0)
    lo_shift = {"band_lo_plus1_" + side: 1, "band_lo_minus1_" + side: -1}.get(mutant, 0)
    vis = visible(sq, sk, mask, device, shift=shift, strict=mutant == "strict_swap", lo_shift=lo_shift)
    if lo is None:
        return vis
    lo = int(lo)
    if mutant == "band_i_end_short" and side == "bwd":
        # per 128-key block, the last 64-row Q block it would visit contributes nothing
        for k0 in range(0, sk, TILE_N):
            q_last = min(k0 + TILE_N - 1, sk - 1) - lo
            if q_last >= 0:
                qb = min(q_last, sq - 1) // TILE_M * TILE_M
                vis[qb:qb + TILE_M, k0:k0 + TILE_N] = False
    if side == "fwd" and mutant in ("band_first_tile_ceil_fwd", "band_wg0_from_wg1_fwd"):
        # the keys below the first tile a warpgroup visits are lost to its 64 rows
        for r in range(0, sq, TILE_M):
            if mutant == "band_first_tile_ceil_fwd":
                t = -(-max(0, r + lo) // TILE_N)
            else:
                t = fwd_first_tile(r + TILE_M if r % TILE_F == 0 else r, lo)
            vis[r:r + TILE_M, :t * TILE_N] = False
    if mutant == "band_need_lo_first_row_bwd" and side == "bwd":
        # on the (key block, Q block) pairs with q0 + lo <= k0 < q0 + 63 + lo the lower edge is not applied
        free = visible(sq, sk, ("band", None, hi), device, shift=shift)
        for k0 in range(0, sk, TILE_N):
            ib, ie = bwd_q_range(k0, sq, sk, lo, None if hi is None else int(hi))
            for i in range(ib, ie):
                q0 = i * TILE_M
                if q0 + lo <= k0 < q0 + TILE_M - 1 + lo:
                    vis[q0:q0 + TILE_M, k0:k0 + TILE_N] = free[q0:q0 + TILE_M, k0:k0 + TILE_N]
    return vis


# --------------------------------------------------------------------------- #
# the document kernels' faults, through their index arithmetic (doc_index)
# --------------------------------------------------------------------------- #
# doc_index's name of each kernel fault of lowp_doc.DOC_MUTANTS, and the side it acts on (None: both)
_DOC_KERNEL_FAULT = {
    "doc_edge_plus1_fwd": ("fwd_edge_plus1", "fwd"), "doc_edge_plus1_bwd": ("bwd_edge_plus1", "bwd"),
    "doc_edge_minus1_fwd": ("fwd_edge_minus1", "fwd"), "doc_edge_minus1_bwd": ("bwd_edge_minus1", "bwd"),
    "doc_range_first_row_fwd": ("range_first_row_only", "fwd"), "doc_i_end_first_key_bwd": ("i_end_first_key", "bwd"),
    "doc_search_lower_bound": ("search_lower_bound", None),
}


def doc_launch(sq, sk, mask):
    """The doc_index restatement of the launch a document mask describes."""
    _, lo, hi, cu, q_pos0, k_pos0, ps = mask
    return di.Launch(sq, sk, hi is not None, 0 if hi is None else hi, lo, cu, q_pos0, k_pos0, ps)


def _doc_kernel_vis(sq, sk, mask, fault, side):
    """Visibility as the doc kernels compute it, with doc_index's ``fault``: the forward's row limits inside its
    warpgroup's tile range, or the backward's Q-block ranges with the staged offsets and the band."""
    L = doc_launch(sq, sk, mask)
    vis = torch.zeros(sq, sk, dtype=torch.bool)
    if side == "fwd":
        for r0 in range(0, sq, 64):
            f, e = L.group_range(r0, fault)
            for a in range(r0, min(r0 + 64, sq)):
                lo, hi = L.row_limits(a, fault)
                lo, hi = max(lo, f * di.BN), min(hi, e * di.BN - 1)
                if lo <= hi:
                    vis[a, lo:hi + 1] = True
        return vis
    c = torch.arange(sk)
    for x in range((sk + di.BWD_N - 1) // di.BWD_N):
        ib, ie = L.q_blocks(x, fault)
        k0 = x * di.BWD_N
        for a in range(ib * di.BWD_M, min(ie * di.BWD_M, sq)):
            lo, hi = L.staged(a, x, fault)
            blk = (c >= k0 + lo) & (c < k0 + hi) & (c >= a + L.lo)
            if L.causal:
                blk &= c <= a + L.off
            vis[a] |= blk
    return vis


def planner_drops_last_key(sq, sk, mask):
    """True when the planner with its last-key fault would drop this launch (``_doc_trim`` taking the keys' last
    document from key sk - 2)."""
    _, _, _, cu, q_pos0, k_pos0, ps = mask
    if sk < 2:
        return False
    d0 = max(di.doc_of(cu, q_pos0), di.doc_of(cu, k_pos0))
    d1 = min(di.doc_of(cu, q_pos0 + ps * (sq - 1)), di.doc_of(cu, k_pos0 + ps * (sk - 2)))
    return d0 > d1


def _doc_vis_for(sq, sk, mask, device, mutant, side):
    """``_vis_for`` of a document mask: the causal mutants act on its band, ``lowp_doc.DOC_MUTANTS`` through the
    kernels' (and the planner's) index arithmetic."""
    if mutant in _DOC_KERNEL_FAULT:
        fault, only = _DOC_KERNEL_FAULT[mutant]
        if only in (None, side):
            return _doc_kernel_vis(sq, sk, mask, fault, side).to(device)
    if mutant == "doc_planner_drop_last_key" and planner_drops_last_key(sq, sk, mask):
        return torch.zeros(sq, sk, dtype=torch.bool, device=device)
    shift = {"causal_plus1_" + side: 1, "causal_minus1_" + side: -1}.get(mutant, 0)
    return visible(sq, sk, mask, device, shift=shift, strict=mutant == "strict_swap")


def lowp_forward(q, k, v, scale, mask=None, key_bias=None, state=None, last=True, mutant=None):
    """One forward chunk with carried state, rounded like ``fwd_chunk_kernel``.

    q [B,Sq,H,D], k/v [B,Sk,Hkv,D] (16-bit); key_bias fp32 [B|1,H,Sk] or None; state ``(o_acc fp32 [B,Sq,H,D],
    lse fp32 [B,H,Sq])`` from the previous chunk or None.  Returns ``(o, lse)``: o in the input dtype when ``last``,
    else the fp32 normalised state the kernel leaves in o_acc.  Rows that see nothing have o = 0 and lse = -inf.
    """
    dtype = q.dtype
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    kk, vv = _kv_heads(k, H, mutant), _kv_heads(v, H, mutant)
    s = _scores_log2(q, kk, scale, key_bias, mutant, "fwd")
    vis = _vis_for(Sq, Sk, mask, q.device, mutant, "fwd")
    if vis is not None:
        s = s.masked_fill(~vis, NEG_INF)
    for j in _drop_keys(Sk, mutant):
        if 0 <= j < Sk:
            s[..., j] = NEG_INF
    m = s.amax(-1)  # [B,H,Sq]
    if state is not None:
        o0 = state[0].float().permute(0, 2, 1, 3)  # [B,H,Sq,D]
        lse0 = state[1].float()
        alive = lse0 != NEG_INF
        m0 = lse0 * LOG2E
        l0 = alive.float() * (4.0 if mutant == "carried_l4" else 1.0)
        if mutant == "dead_revive_stale_m":
            m0 = torch.where(alive, m0, torch.zeros_like(m0))
            l0 = torch.ones_like(l0)
        m = torch.maximum(m, m0)
    msafe = torch.where(m == NEG_INF, torch.zeros_like(m), m)
    p = torch.exp2(s - msafe.unsqueeze(-1))
    l = p.sum(-1)
    o = torch.einsum("bhqk,bhkd->bhqd", _round(p, dtype), vv.float().permute(0, 2, 1, 3))
    if state is not None:
        f = torch.exp2(m0 - msafe)
        l = l + l0 * f
        o = o + o0 * f.unsqueeze(-1)
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    o = (o * inv.unsqueeze(-1)).permute(0, 2, 1, 3).contiguous()
    lse = torch.where(l > 0, (m + torch.log2(l)) * LN2, torch.full_like(l, NEG_INF))
    return (o.to(dtype) if last else o), lse


def lowp_backward(q, k, v, do, o, lse, scale, mask=None, key_bias=None, mutant=None):
    """One backward chunk, rounded like ``delta_kernel`` + ``bwd_chunk_kernel``.

    o: the 16-bit forward output, lse: the final fp32 lse (-inf: the row saw nothing, P = 0).
    Returns fp32 ``(dq [B,Sq,H,D], dk [B,Sk,Hkv,D], dv [B,Sk,Hkv,D])`` partials of this chunk.
    """
    dtype = q.dtype
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    kk, vv = _kv_heads(k, H, mutant), _kv_heads(v, H, mutant)
    delta = (o.float() * do.float()).sum(-1).permute(0, 2, 1)  # [B,H,Sq]
    s = _scores_log2(q, kk, scale, key_bias, mutant, "bwd")
    lse2 = torch.where(lse == NEG_INF, torch.full_like(lse, float("inf")), lse.float()) * LOG2E
    p = torch.exp2(s - lse2.unsqueeze(-1))
    vis = _vis_for(Sq, Sk, mask, q.device, mutant, "bwd")
    if vis is not None:
        p = p.masked_fill(~vis, 0.0)
    for j in _drop_keys(Sk, mutant):
        if 0 <= j < Sk:
            p[..., j] = 0.0
    p_dv = _round(p, dtype)
    if mutant == "dv_missing_q_block" and mask is not None:
        # per 128-key block, skip the first 64-row Q block it would visit
        off = int(mask[1])
        for k0 in range(0, Sk, 128):
            qb = max(0, k0 - off) // 64 * 64
            p_dv[..., qb:qb + 64, k0:k0 + 128] = 0.0
    dv = torch.einsum("bhqk,bqhd->bkhd", p_dv, do.float())
    dp = torch.einsum("bqhd,bkhd->bhqk", do.float(), vv.float())
    ds = _round(p * (dp - delta.unsqueeze(-1)), dtype)
    ds_q = ds
    if mutant == "dq_missing_key_block":
        kb = 128 if Sk > 128 else 0
        ds_q = ds.clone()
        ds_q[..., kb:kb + 128] = 0.0
    dq = torch.einsum("bhqk,bkhd->bqhd", ds_q, kk.float()) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q.float()) * (1.0 if mutant == "dk_no_scale" else scale)
    return dq, _group_sum(dk, Hkv), _group_sum(dv, Hkv)


# --------------------------------------------------------------------------- #
# ALiBi: fwd_alibi_kernel / bwd_alibi_kernel (csrc/fwd_sm90.cuh, csrc/bwd_sm90.cuh)
# --------------------------------------------------------------------------- #
# ``lowp_alibi_forward`` / ``lowp_alibi_backward`` restate what the ALiBi kernels compute for ``alibi = (slopes [B, H],
# dist0, pstride)``, rounding where the kernels round (DESIGN 5.1b) and otherwise as the plain model does:
#
# * distances: row a and key c are ``d = pstride (a - c) + dist0`` apart, an exact int64; each row's reference ``dref``
#   is its smallest |d| over the chunk's keys (``alibi_dref``), lowered under a live carried state of lse m0 (log2
#   units) to the truncated fp32 ``cap = max(0, -m0) / slope2`` when that is smaller (``alibi_carried_ref``);
# * forward: the fp32 log2 scores get ``fp32(-slope2 (|d| - dref))`` (slope2 = slope log2(e) in fp32); the carried
#   state enters as ``m = fma(slope2, dref, m0)``; lse is ``(m + log2 l - slope2 dref) ln2``;
# * backward, per tile of 64 rows x 128 keys from k0 (both kernels classify such tiles): on a tile where d has one
#   sign s the loader's row statistic is ``fma(slope2, fp32(s (pstride (q - k0) + dist0)), fp32(lse log2(e)))`` and
#   the exponent adds the per-key term ``s slope2 pstride (c - k0)``; on a tile across d = 0 it adds ``-slope2 |d|``.
#
# Slopes are indexed by the query head, under GQA too.  The faults of ``lowp_alibi.ALIBI_MUTANTS`` act here.
F32 = torch.float32
LOG2E_F = torch.tensor(LOG2E, dtype=F32)
LN2_F = torch.tensor(LN2, dtype=F32)


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
    kk, vv = _kv_heads(k, H), _kv_heads(v, H)
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
    s = raw * _scale_log2(scale) + bias2
    vis = visible(Sq, Sk, mask, dev)
    if vis is not None:
        s = s.masked_fill(~vis, NEG_INF)
    m = s.amax(-1)
    if state is not None:
        m_c = _fma(slope2.view(B, H, 1).expand(B, H, Sq), dref_f, m0)  # m0 + slope2 dref: the row's frame
        m = torch.where(alive, torch.maximum(m, m_c), m)
    msafe = torch.where(m == NEG_INF, torch.zeros_like(m), m)
    p = torch.exp2(s - msafe.unsqueeze(-1))
    l = p.sum(-1)
    o = torch.einsum("bhqk,bhkd->bhqd", _round(p, dtype), vv.float().permute(0, 2, 1, 3))
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
    kk, vv = _kv_heads(k, H), _kv_heads(v, H)
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
    p = torch.exp2(_fma(raw, torch.tensor(_scale_log2(scale), dtype=F32), x0))
    vis = visible(Sq, Sk, mask, dev)
    if vis is not None:
        p = p.masked_fill(~vis, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", _round(p, dtype), do.float())
    dp = torch.einsum("bqhd,bkhd->bhqk", do.float(), vv.float())
    ds = _round(p * (dp - delta.unsqueeze(-1)), dtype)
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk.float()) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q.float()) * scale
    return dq, _group_sum(dk, Hkv), _group_sum(dv, Hkv)


# --------------------------------------------------------------------------- #
# chains of chunks: the model and the fp64 oracle side by side
# --------------------------------------------------------------------------- #
def lowp_chain(q, ks, vs, do, scale, masks, biases=None, mutant=None, alibis=None, lse_bwd=None, info=None):
    """Forward over K/V chunks ``ks[c], vs[c]`` (mask ``masks[c]``, key bias ``biases[c]`` or ALiBi ``alibis[c] =
    (slopes, dist0, pstride)``) with the fp32 state carried between chunks, then the backward of every chunk against
    the final (O, lse).  ``info``: as in ``lowp_alibi_forward``.

    ``lse_bwd``: the fp32 lse the backward reads (default: the model's own).  An ALiBi kernel test passes the kernels'
    own: far from d = 0 the backward turns the fp32 rounding of lse itself (ulp(slope dref), DESIGN 5.1b) into an error
    of P that the model reproduces only from the same lse; the lse is held to the oracle on its own.
    Returns dict(o, lse, states=[(o_acc, lse) after each non-last chunk], dq, dk=[per chunk], dv=[per chunk])."""
    n = len(ks)
    biases = biases or [None] * n
    alibis = alibis or [None] * n
    state, states = None, []
    for c in range(n):
        if alibis[c] is None:
            o, lse = lowp_forward(q, ks[c], vs[c], scale, masks[c], biases[c], state, last=c == n - 1, mutant=mutant)
        else:
            o, lse = lowp_alibi_forward(q, ks[c], vs[c], scale, masks[c], alibis[c], state, last=c == n - 1,
                                        mutant=mutant, info=info)
        if c < n - 1:
            state = (o, lse)
            states.append(state)
    lb = lse if lse_bwd is None else lse_bwd.to(q.device)
    dq = torch.zeros(q.shape, device=q.device, dtype=torch.float32)
    dks, dvs = [], []
    for c in range(n):
        if alibis[c] is None:
            dqc, dk, dv = lowp_backward(q, ks[c], vs[c], do, o, lb, scale, masks[c], biases[c], mutant=mutant)
        else:
            dqc, dk, dv = lowp_alibi_backward(q, ks[c], vs[c], do, o, lb, scale, masks[c], alibis[c], mutant=mutant)
        dq += dqc
        dks.append(dk)
        dvs.append(dv)
    return dict(o=o, lse=lse, states=states, dq=dq, dk=dks, dv=dvs)


def oracle_chain(q, ks, vs, do, scale, masks, biases=None, alibis=None, device="cpu"):
    """The same chain in fp64 with ``mask_oracle`` (on ``device``, the CPU by default), on the same 16-bit inputs;
    ALiBi enters as each chunk's pair bias (``mask_oracle.chunk_bias``)."""
    n = len(ks)
    dev = lambda t: None if t is None else t.detach().to(device)  # noqa: E731
    q, do = dev(q), dev(do)
    H, Hkv = q.shape[2], ks[0].shape[2]
    kx = [_kv_heads(dev(k), H) for k in ks]
    vx = [_kv_heads(dev(v), H) for v in vs]
    biases = [dev(b) for b in biases] if biases else [None] * n
    if alibis:
        biases = [b if a is None else mo.chunk_bias((dev(a[0]), a[1], a[2]), q.shape[1], kx[c].shape[1])
                  for c, (a, b) in enumerate(zip(alibis, biases))]
    o, lse, states = None, None, []
    for c in range(n):
        o, lse = mo.chunk_forward(q, kx[c], vx[c], o, lse, scale, masks[c], bias=biases[c])
        if c < n - 1:
            states.append((o, lse))
    delta = orc.compute_delta(o, do)
    lse_b = torch.where(torch.isinf(lse), torch.full_like(lse, float("inf")), lse)  # dead rows: P = 0
    dq = torch.zeros(q.shape, dtype=torch.float64, device=q.device)
    dks, dvs = [], []
    for c in range(n):
        dqc, dk, dv = mo.chunk_backward(do, q, kx[c], vx[c], delta, lse_b, scale, masks[c], bias=biases[c])
        dq += dqc
        dks.append(_group_sum(dk, Hkv))
        dvs.append(_group_sum(dv, Hkv))
    return dict(o=o, lse=lse, states=states, dq=dq, dk=dks, dv=dvs,
                **error_scales(q, kx, vx, do, o, delta, lse_b, scale, masks, biases, Hkv))


def error_scales(q, kx, vx, do, o, delta, lse_b, scale, masks, biases, Hkv):
    """The comparator's error scales of one fp64 chain (``oracle_chain``): dict(mag, rss, e32, sums).  Tensors on one
    device; kx / vx per chunk at the query heads; lse_b the final lse with +inf for dead rows; ``biases[c]``: None, a
    key bias [B|1,H,Sk] or a pair bias [B,H,Sq,Sk], in natural units.  ``sums``: the ``error_sums`` the scales are
    finished from (``finish_scales``)."""
    sums = error_sums(q, kx, vx, do, o, delta, lse_b, scale, masks, biases)
    return dict(mag=magnitudes(q, kx, vx, do, scale), sums=sums,
                **finish_scales(sums, o, Hkv, [k.shape[1] for k in kx]))


def error_sums(q, kx, vx, do, o, delta, lse_b, scale, masks, biases):
    """The additive parts of ``error_scales``: per row (fp64 [B,Sq,H]) and, per chunk, per key and query head (fp64
    [B,Sk,H]) sums over the pairs a chain sees.  A problem cut into row blocks adds the per-key sums of its blocks."""
    n = len(kx)
    # Per gradient row, two error scales no 16-bit model run reproduces by itself:
    # rss: the root sum of squares of the row's terms (P V for O, P dO for dV, dS K scale for dQ, dS Q scale for dK).
    #   A 16-bit rounding moves each term by at most u/2 of itself, so where a row's terms cancel (sum_k dS = 0
    #   exactly) or one term dominates, one model run can happen to land near the truth while the kernel does not.
    #   delta comes from the 16-bit O, whose rounding moves delta by ~u sqrt(sum_d (O_d dO_d)^2) and every dS of the
    #   row by P times that: in a peaky row this term, not the rounding of dS, dominates dQ and dK (for dK the
    #   rows' shifts are added coherently, an upper bound: ``dk_coh`` is that sum, squared in ``finish_scales``).
    # e32: dS = P (dP - delta) with dP from fp32 tensor-core accumulation and delta from a separate fp32 sum keeps
    #   ~2^-23 sum_d |dO_d V_d| of rounding per element, which reaches dQ through |K| and dK through |Q|.
    z = lambda: torch.zeros(q.shape[:3], dtype=torch.float64, device=q.device)  # noqa: E731
    out = dict(o=z(), dq=z(), dq_coh=z(), e32_dq=z(), dk=[], dk_coh=[], dv=[], e32_dk=[])
    qd, dod = q.double(), do.double()
    n2 = lambda t: t.double().pow(2).sum(-1)  # noqa: E731  [B,S,H] squared row norms
    dd = n2(o.double() * dod).sqrt().permute(0, 2, 1)  # [B,H,Sq]
    for c in range(n):
        kd, vd = kx[c].double(), vx[c].double()
        s = torch.einsum("bqhd,bkhd->bhqk", qd, kd) * scale
        if biases[c] is not None:
            b = biases[c].double()
            s = s + (b if b.dim() == 4 else b.unsqueeze(2))
        p = torch.exp(s - lse_b.unsqueeze(-1))
        del s
        vis = visible(q.shape[1], kd.shape[1], masks[c], q.device)
        if vis is not None:
            p = p.masked_fill(~vis, 0.0)
        ds = p * (torch.einsum("bqhd,bkhd->bhqk", dod, vd) - delta.unsqueeze(-1)) * scale
        out["o"] += torch.einsum("bhqk,bkh->bqh", p * p, n2(vd))
        pd = p * dd.unsqueeze(-1) * abs(scale)  # [B,H,Sq,Sk]: the dS shift of one unit of delta rounding
        out["dq"] += torch.einsum("bhqk,bkh->bqh", ds * ds, n2(kd))
        out["dq_coh"] += torch.einsum("bhqk,bkh->bqh", pd, kd.norm(dim=-1))
        out["dk"].append(torch.einsum("bhqk,bqh->bkh", ds * ds, n2(qd)))
        out["dk_coh"].append(torch.einsum("bhqk,bqh->bkh", pd, qd.norm(dim=-1)))
        out["dv"].append(torch.einsum("bhqk,bqh->bkh", p * p, n2(dod)))
        del ds, pd
        w = 2.0 ** -23 * abs(scale) * p * torch.einsum("bqhd,bkhd->bhqk", dod.abs(), vd.abs())
        out["e32_dq"] += torch.einsum("bhqk,bkh->bqh", w, kd.norm(dim=-1))
        out["e32_dk"].append(torch.einsum("bhqk,bqh->bkh", w, qd.norm(dim=-1)))
    return out


def finish_scales(sums, o, Hkv, sks):
    """dict(rss, e32) of ``error_sums`` (dK / dV per key, the chunks' keys in order, their K/V heads summed)."""
    n2 = lambda t: t.double().pow(2).sum(-1)  # noqa: E731
    g = lambda t: _group_sum(t.unsqueeze(-1), Hkv)[..., 0]  # noqa: E731  [B,Sk,H] -> [B,Sk,Hkv]
    rss = dict(o=(sums["o"] + n2(o)).sqrt(), dq=(sums["dq"] + sums["dq_coh"].pow(2)).sqrt(),
               dk=torch.cat([g(a + c.pow(2)) for a, c in zip(sums["dk"], sums["dk_coh"])], 1).sqrt(),
               dv=torch.cat([g(a) for a in sums["dv"]], 1).sqrt())
    return dict(rss=rss, e32=dict(dq=sums["e32_dq"], dk=torch.cat([g(a) for a in sums["e32_dk"]], 1)))


def magnitudes(q, kx, vx, do, scale):
    """The size of one key's contribution to a gradient row, before any cancellation (the comparator's floor):
    dict(dq, dk, dv) from the largest row norms of the inputs (kx / vx: the chunks' K / V)."""
    nrm = lambda ts: max(float(t.double().norm(dim=-1).max()) for t in ts)  # noqa: E731
    nq, ndo, nk, nv = nrm([q]), nrm([do]), nrm(kx), nrm(vx)
    return dict(dq=abs(scale) * ndo * nv * nk, dk=abs(scale) * ndo * nv * nq, dv=ndo)


def scores_absmax(q, ks, scale, masks, biases=None, device="cpu"):
    """[B,H,Sq]: per row, the largest ``sum_d |q_d k_d| scale + |bias|`` over the keys the row sees in any chunk --
    the magnitude the fp32 score arithmetic works at, which bounds its rounding error.  ``biases[c]``: None, a key
    bias [B|1,H,Sk] or a pair bias [B,H,Sq,Sk].  Computed on ``device``."""
    n = len(ks)
    biases = biases or [None] * n
    q = q.detach().to(device).double().abs()
    H = q.shape[2]
    out = torch.zeros(q.shape[0], H, q.shape[1], dtype=torch.float64, device=q.device)
    for c in range(n):
        k = _kv_heads(ks[c].detach().to(device), H).double().abs()
        a = torch.einsum("bqhd,bkhd->bhqk", q, k) * abs(scale)
        pair = biases[c] is not None and biases[c].dim() == 4
        if biases[c] is not None:
            bb = biases[c].detach().to(device).double().abs()
            bb = torch.where(torch.isinf(bb), torch.zeros_like(bb), bb)
            a = a + (bb if pair else bb.unsqueeze(2))
        vis = visible(q.shape[1], k.shape[1], masks[c], q.device)
        if vis is not None:
            a = a.masked_fill(~vis, 0.0)
        if biases[c] is not None:
            inf = torch.isinf(biases[c].detach().to(device))
            a = a.masked_fill((inf if pair else inf.unsqueeze(2)).expand_as(a), 0.0)
        out = torch.maximum(out, a.amax(-1))
    return out


# --------------------------------------------------------------------------- #
# the comparator
# --------------------------------------------------------------------------- #
# Global: max|got - ref| <= A * max|model - ref| + FLOOR * mag (+ max(extra), below).
# Per (b, s, h) row of length D: |got - ref| <= B * |model - ref| + C * u * rss + FLOOR * mag + extra, where rss is
# the root sum of squares of the row's terms (default |ref|) and extra (dQ, dK) the fp32 bound e32, both from
# ``oracle_chain``; the global bound adds max(extra).
# mag is the size of one unit of the output before any cancellation (default: the largest row norm of ref; for the
# gradients ``oracle_chain`` derives it from the input norms): where the exact result cancels to zero -- dQ and dK
# of a row or key with a single visible partner, whose dS = P (dP - delta) is exactly zero -- the kernels are left
# with the fp32 rounding of dP - delta, which no 16-bit model reproduces.
# lse: |got - ref| <= LSE_A * 2^-23 * (|ref| + scores_absmax), -inf exactly where the reference is -inf.
# Set from the H100 calibration of tests/test_gpu_tile_edges.py so that the kernels use at most half of every bound
# (WORST; test_report_worst_ratios there prints it).  The same constants serve bf16 and fp16: u carries the dtype.
A = 3.0
B = 4.0
C = 2.0
FLOOR = 2.0 ** -20
LSE_A = 4.0

# worst bound usage seen in this process, error / bound (the check passes at <= 1):
# {(output, dtype name): ((global usage, case), (worst row usage, case))}
WORST: dict = {}


def _note(name, dt, glob, row):
    key = (name.split("[")[0], dt)
    case = name[name.find("[") + 1:-1] if "[" in name else name
    g0, r0 = WORST.get(key, ((0.0, ""), (0.0, "")))
    WORST[key] = (max(g0, (glob, case)), max(r0, (row, case)))


def assert_within_model(name, got, ref, model, dtype, mag=None, extra=None, rss=None):
    """``got`` (kernel), ``ref`` (fp64 oracle) and ``model`` (lowp_*) of one output [B,S,H,D]; see the constants."""
    got, ref, model = (t.detach().double().cpu() for t in (got, ref, model))
    assert got.shape == ref.shape == model.shape, (name, got.shape, ref.shape, model.shape)
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} non-finite values"
    u = unit_roundoff(dtype)
    err, merr = (got - ref).abs(), (model - ref).abs()
    en, mn, rn = (got - ref).norm(dim=-1), (model - ref).norm(dim=-1), ref.norm(dim=-1)
    if mag is None:
        mag = float(rn.max()) if rn.numel() else 0.0
    floor = FLOOR * mag
    extra = torch.zeros_like(en) if extra is None else extra.detach().double().cpu()
    rss = rn if rss is None else rss.detach().double().cpu()
    tiny = torch.finfo(torch.float64).tiny
    g_err, g_model = float(err.max()), float(merr.max())
    g_bound = A * g_model + floor + float(extra.max())
    g_use = g_err / max(g_bound, tiny) if g_err > 0 else 0.0
    row_bound = (B * mn + C * u * rss + floor + extra).clamp(min=tiny)
    row_use = torch.where(en > 0, en / row_bound, torch.zeros_like(en))
    _note(name, str(dtype).replace("torch.", ""), g_use, float(row_use.max()))
    assert g_use <= 1.0, (
        f"{name}: max|got-ref| {g_err:.3e} > {A} x max|model-ref| {g_model:.3e} + floor {floor:.1e} + "
        f"fp32 term {float(extra.max()):.1e} "
        f"(at {tuple(int(i) for i in torch.unravel_index(err.argmax(), err.shape))})")
    bad = row_use > 1.0
    if bad.any():
        idx = bad.nonzero()
        worst = tuple(int(i) for i in torch.unravel_index(row_use.argmax(), row_use.shape))
        raise AssertionError(
            f"{name}: {int(bad.sum())} of {bad.numel()} (b, s, h) rows outside the model bound, e.g. rows "
            f"(b, s, h) {[tuple(r) for r in idx[:8].tolist()]}; worst {worst}: |got-ref| {float(en[worst]):.3e}, "
            f"|model-ref| {float(mn[worst]):.3e}, |ref| {float(rn[worst]):.3e}")


def assert_lse(name, got, ref, absmax):
    """lse [B,H,S] (fp32 kernel vs fp64 oracle); ``absmax`` from ``scores_absmax``."""
    got, ref, absmax = (t.detach().double().cpu() for t in (got, ref, absmax))
    dead = torch.isinf(ref) & (ref < 0)
    assert not torch.isnan(got).any(), f"{name}: NaN in lse"
    assert torch.equal(torch.isinf(got) & (got < 0), dead), (
        f"{name}: lse is -inf at {int((torch.isinf(got) & (got < 0)).sum())} rows, the oracle at {int(dead.sum())}")
    g, r, a = got[~dead], ref[~dead], absmax[~dead]
    if g.numel() == 0:
        return
    tol = 2.0 ** -23 * (r.abs() + a)
    ratio = float(((g - r).abs() / tol.clamp(min=torch.finfo(torch.float64).tiny)).max())
    _note(name, "fp32", ratio / LSE_A, ratio / LSE_A)
    assert ratio <= LSE_A, f"{name}: |lse - ref| reaches {ratio:.2f} x 2^-23 (|ref| + scores_absmax), limit {LSE_A}"


def uniform_closed_form(vs, masks, sq):
    """q = 0 and no bias: every visible key has the same score, so O is the mean of the visible V rows and
    lse = log(#visible).  vs: the chunks' V [B,Sk,H,D] (already at the query heads); returns fp64
    (o [B,Sq,H,D], lse [Sq])."""
    num, n = 0.0, torch.zeros(sq, dtype=torch.float64)
    for v, m in zip(vs, masks):
        v = v.detach().cpu().double()
        vis = visible(sq, v.shape[1], m)
        w = torch.ones(sq, v.shape[1], dtype=torch.float64) if vis is None else vis.double()
        num = num + torch.einsum("qk,bkhd->bqhd", w, v)
        n += w.sum(-1)
    o = num / n.clamp(min=1).view(1, sq, 1, 1)
    lse = torch.where(n > 0, n.log(), torch.full_like(n, NEG_INF))
    return o, lse


def assert_chain_within_model(name, got, ref, model, dtype, absmax_prefix):
    """Every output of a chain (``lowp_chain`` / ``oracle_chain`` dicts): the fp32 state after each non-last chunk,
    O, lse, dQ and the per-chunk dK, dV.  ``absmax_prefix[c]``: ``scores_absmax`` over chunks 0..c."""
    for c, (g, r, m) in enumerate(zip(got["states"], ref["states"], model["states"])):
        assert_within_model(f"o_acc[{name} chunk {c}]", g[0], r[0], m[0], dtype)
        assert_lse(f"lse_state[{name} chunk {c}]", g[1], r[1], absmax_prefix[c])
    r = ref
    assert_within_model(f"o[{name}]", got["o"], r["o"], model["o"], dtype, rss=r["rss"]["o"])
    assert_lse(f"lse[{name}]", got["lse"], r["lse"], absmax_prefix[-1])
    assert_within_model(f"dq[{name}]", got["dq"], r["dq"], model["dq"], dtype, r["mag"]["dq"], r["e32"]["dq"],
                        r["rss"]["dq"])
    cat = lambda d, k: torch.cat([t.detach().cpu().double() for t in d[k]], dim=1)  # noqa: E731
    assert_within_model(f"dk[{name}]", cat(got, "dk"), cat(r, "dk"), cat(model, "dk"), dtype, r["mag"]["dk"],
                        r["e32"]["dk"], r["rss"]["dk"])
    assert_within_model(f"dv[{name}]", cat(got, "dv"), cat(r, "dv"), cat(model, "dv"), dtype, r["mag"]["dv"],
                        rss=r["rss"]["dv"])


def assert_api_within_model(name, got, ref, model, dtype, absmax=None):
    """What the public API returns for one call -- ``got``: dict(o, dq, dk, dv) [B,S,H,D] and, checked when
    ``absmax`` (``scores_absmax``) is given, lse [B,H,S] -- against ``oracle_chain`` / ``lowp_chain`` of the same
    problem.  The API returns 16-bit gradients, so the model's fp32 gradients are rounded to 16 bit first."""
    rnd = lambda t: t.to(dtype).float()  # noqa: E731
    cat = lambda d, k: torch.cat([t.detach().cpu().double() for t in d[k]], dim=1)  # noqa: E731
    r = ref
    assert_within_model(f"o[{name}]", got["o"], r["o"], model["o"], dtype, rss=r["rss"]["o"])
    if absmax is not None:
        assert_lse(f"lse[{name}]", got["lse"], r["lse"], absmax)
    assert_within_model(f"dq[{name}]", got["dq"], r["dq"], rnd(model["dq"]), dtype, r["mag"]["dq"], r["e32"]["dq"],
                        r["rss"]["dq"])
    assert_within_model(f"dk[{name}]", got["dk"], cat(r, "dk"), rnd(cat(model, "dk")), dtype, r["mag"]["dk"],
                        r["e32"]["dk"], r["rss"]["dk"])
    assert_within_model(f"dv[{name}]", got["dv"], cat(r, "dv"), rnd(cat(model, "dv")), dtype, r["mag"]["dv"],
                        rss=r["rss"]["dv"])


# --------------------------------------------------------------------------- #
# the tile-edge sweep (tests/test_gpu_tile_edges.py runs it on the kernels, tests/test_lowp_model.py on the model)
# --------------------------------------------------------------------------- #
# Forward tiles are 128 Q rows x 128 keys; backward tiles 128 keys x 64 Q rows.  A case: Sq query rows against a
# chain of K/V chunks (Sk, causal offset or None), the softmax scale ("d": D^-0.5), a score distribution, a key
# bias kind, batch / heads, the layout the kernels see ("flash" [B,S,H,D], "normal" [B,H,S,D], "bstride": x[::2] of
# a batch twice as large) and an input amplitude.
_DT = (torch.bfloat16, torch.float16)
_OFFSETS = lambda sq, sk: [-sk, -129, -128, -65, -64, -63, -1, 0, 1, 63, 64, 65, 127, 128, 129, sk - sq, sk]  # noqa


def _case(sq, chunks, D=128, dtype=torch.bfloat16, scale="d", dist="randn", bias=None, B=1, H=2, Hkv=None,
          layout="flash", amp=1.0, tag=""):
    if len(chunks) > 3:  # long chains: number of chunks, total keys, offset of the first chunk
        ch = f"{len(chunks)}chunks{sum(sk for sk, _ in chunks)}" + ("" if chunks[0][1] is None else f"@{chunks[0][1]}")
    else:
        ch = "+".join(f"{sk}" + ("" if off is None else f"@{off}") for sk, off in chunks)
    name = f"{tag}q{sq}_k{ch}_d{D}_{'bf16' if dtype == torch.bfloat16 else 'fp16'}_s{scale}_{dist}"
    if bias:
        name += f"_bias-{bias}"
    if B != 1 or H != 2 or Hkv:
        name += f"_B{B}H{H}kv{Hkv or H}"
    if layout != "flash":
        name += f"_{layout}"
    if amp != 1.0:
        name += f"_x{amp:g}"
    return dict(id=name, sq=sq, chunks=list(chunks), D=D, dtype=dtype, scale=scale, dist=dist, bias=bias, B=B, H=H,
                Hkv=Hkv or H, layout=layout, amp=amp)


def _sweep():
    cases = []
    # every Sq in {1, 63, 64, 65, 127, 128, 129, 255, 257, 383} and Sk in {1, 2, 63, 127, 128, 129, 255, 256, 257, 513}
    pairs = [(1, 513), (63, 129), (64, 1), (65, 127), (127, 2), (128, 257), (129, 63), (255, 128), (257, 255),
             (383, 256), (1, 1), (129, 129), (257, 513), (65, 2)]
    for i, (sq, sk) in enumerate(pairs):
        for j, (D, dt) in enumerate([(64, _DT[0]), (64, _DT[1]), (128, _DT[0]), (128, _DT[1])]):
            cases.append(_case(sq, [(sk, None)], D, dt))
        D, dt = [(64, _DT[0]), (128, _DT[1]), (128, _DT[0]), (64, _DT[1])][i % 4]
        cases.append(_case(sq, [(sk, sk - sq)], D, dt))  # bottom-right causal
    # causal offsets one key either side of every forward (128) and backward (64) tile edge, both signs
    for sq, sk in [(255, 257), (129, 513)]:
        for i, off in enumerate(_OFFSETS(sq, sk)):
            D, dt = [(128, _DT[0]), (64, _DT[1]), (64, _DT[0]), (128, _DT[1])][i % 4]
            cases.append(_case(sq, [(sk, off)], D, dt))
    # softmax scales x score distributions
    for i, scale in enumerate([0.01, "d", 0.3, 1.0]):
        for j, dist in enumerate(["randn", "rising", "last_tile", "zero_q"]):
            D, dt = [(128, _DT[0]), (64, _DT[1]), (128, _DT[1]), (64, _DT[0])][(i + j) % 4]
            sq, sk = (129, 257) if j % 2 == 0 else (255, 513)
            off = None if (i + j) % 2 == 0 else sk - sq
            cases.append(_case(sq, [(sk, off)], D, dt, scale=scale, dist=dist))
    # carried state: chains of 2, 5 and 16 chunks (views of one causal problem: offset = q_start - k_start)
    def causal_chain(sq, sizes, q_start):
        out, k0 = [], 0
        for sk in sizes:
            out.append((sk, q_start - k0))
            k0 += sk
        return out
    for D, dt in [(128, _DT[0]), (64, _DT[1])]:
        cases.append(_case(129, [(128, None), (129, None)], D, dt))
        cases.append(_case(129, causal_chain(129, [128, 129], 128), D, dt))
        cases.append(_case(255, [(63, None), (127, None), (1, None), (129, None), (255, None)], D, dt))
        cases.append(_case(255, causal_chain(255, [128] * 5, 640 - 255), D, dt))
        cases.append(_case(129, [(64, None)] * 16, D, dt))
        cases.append(_case(129, causal_chain(129, [64] * 16, 1024 - 129), D, dt))
        # the first chunk leaves every row (offset <= -Sq) or the first 64 rows dead; later chunks revive them
        cases.append(_case(129, [(128, -129), (128, 128), (129, 0)], D, dt, tag="dead1st_"))
        cases.append(_case(129, [(128, -64), (257, 200)], D, dt, tag="dead1st_"))
        cases.append(_case(65, [(1, -65), (127, -1), (63, 64), (2, 70), (255, 127)], D, dt, tag="dead1st_"))
    cases.append(_case(257, causal_chain(257, [64] * 16, 1024 - 257), 128, _DT[0], scale=1.0, dist="rising"))
    # key bias
    for D, dt in [(128, _DT[0]), (64, _DT[1])]:
        cases.append(_case(129, [(257, None)], D, dt, bias="randn"))
        cases.append(_case(129, [(257, 128)], D, dt, bias="randn"))
        cases.append(_case(127, [(383, None)], D, dt, bias="tile_inf"))
        cases.append(_case(255, [(257, None)], D, dt, bias="edge_inf"))
        cases.append(_case(129, [(257, 128)], D, dt, bias="edge_inf"))
        cases.append(_case(129, [(255, None)], D, dt, bias="bcast", B=2))
        cases.append(_case(129, [(129, 0)], D, dt, bias="dead_rows"))
        cases.append(_case(65, [(128, None)], D, dt, bias="head_dead"))
        cases.append(_case(129, [(128, -64), (129, 64)], D, dt, bias="randn", tag="chain_"))
    # layouts and grouped-query attention
    for D, dt in [(128, _DT[1]), (64, _DT[0])]:
        cases.append(_case(129, [(257, 128)], D, dt, B=2, layout="bstride"))
        cases.append(_case(255, [(129, None)], D, dt, B=2, layout="bstride", bias="randn"))
        cases.append(_case(129, [(257, 65)], D, dt, layout="normal"))
        cases.append(_case(65, [(128, None), (63, 64)], D, dt, layout="normal"))
        for hkv in (4, 2, 1):
            cases.append(_case(129, [(257, 127)], D, dt, H=4, Hkv=hkv))
        cases.append(_case(255, [(129, -63)], D, dt, H=4, Hkv=2, bias="randn", layout="normal"))
    # fp16 range: inputs x 4
    for D in (64, 128):
        cases.append(_case(129, [(513, None)], D, _DT[1], amp=4.0))
        cases.append(_case(255, [(257, 1)], D, _DT[1], scale=1.0, amp=4.0))
        cases.append(_case(129, causal_chain(129, [128, 129], 128), D, _DT[1], amp=4.0))
    ids = [c["id"] for c in cases]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    return cases


SWEEP = _sweep()


def make_inputs(case, device="cpu"):
    """The case's 16-bit inputs in the logical flash layout, on ``device``:
    dict(q, ks, vs, do, scale, masks, biases)."""
    import zlib
    g = torch.Generator().manual_seed(zlib.crc32(case["id"].encode()))
    B, H, Hkv, D, sq, dt, amp = case["B"], case["H"], case["Hkv"], case["D"], case["sq"], case["dtype"], case["amp"]
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float32)  # noqa: E731
    e = torch.ones(D) / D ** 0.5  # a direction every query shares with the keys it favours
    q = rn(B, sq, H, D)
    do = rn(B, sq, H, D)
    ks, vs, k0 = [], [], 0
    n_total = sum(sk for sk, _ in case["chunks"])
    for sk, _ in case["chunks"]:
        k, v = rn(B, sk, Hkv, D), rn(B, sk, Hkv, D)
        pos = torch.arange(k0, k0 + sk, dtype=torch.float32)
        if case["dist"] == "rising":  # every 128-key tile scores higher than the one before
            k = 0.5 * k + ((pos // 128 + 1) * 1.0).view(1, sk, 1, 1) * e
        elif case["dist"] == "last_tile":  # the row maximum sits in the last, ragged tile of the last chunk
            last = pos >= (n_total - 1) // 128 * 128
            k = 0.3 * k + last.float().view(1, sk, 1, 1) * 3.0 * e
        ks.append(k)
        vs.append(v)
        k0 += sk
    if case["dist"] == "rising":
        q = 0.5 * q + 4.0 * e
    elif case["dist"] == "last_tile":
        q = 0.3 * q + 3.0 * e
    elif case["dist"] == "zero_q":
        q = torch.zeros_like(q)
    biases = []
    for sk, _ in case["chunks"]:
        kind = case["bias"]
        if kind is None:
            biases.append(None)
            continue
        b = 2.0 * rn(1 if kind == "bcast" else B, H, sk)
        if kind == "tile_inf":
            b[..., 128:256] = NEG_INF
        elif kind == "edge_inf":
            for j in (127, 128, sk - 1):
                if j < sk:
                    b[..., j] = NEG_INF
        elif kind == "dead_rows":  # with the causal diagonal: rows 0..63 see only these keys
            b[..., :64] = NEG_INF
        elif kind == "head_dead":  # every key of the last query head
            b[:, -1] = NEG_INF
        if kind == "bcast":
            b = b.expand(B, H, sk)
        biases.append(b.to(device))
    scale = D ** -0.5 if case["scale"] == "d" else float(case["scale"])
    cvt = lambda t: (amp * t).to(dt).to(device)  # noqa: E731
    return dict(q=cvt(q), ks=[cvt(k) for k in ks], vs=[cvt(v) for v in vs], do=cvt(do), scale=scale,
                masks=[None if off is None else ("causal_offset", off) for _, off in case["chunks"]], biases=biases)
