"""fp64 CPU oracle of attention under every mask and bias the kernels take, for the tests only.

``oracle/attention_oracle.py`` states the reference's masks (none / causal / causal offset); this module adds, in the
same conventions (flash layout [B, S, H, D], math in fp64), what the window, ALiBi and packed-document tests need:

* ``mask_of``: one chunk's kernel mask -- None, ``("causal_offset", off)`` (key b visible to row a iff b <= a + off),
  ``("band", lo, hi)`` (iff a + lo <= b <= a + hi, None for an open side) or ``("doc", lo, hi, cu, q_pos0, k_pos0,
  pstride)`` (the band, and row a at position q_pos0 + pstride a sees key b at k_pos0 + pstride b only inside one
  document ``[cu[d], cu[d + 1])``);
* ``chunk_forward`` / ``chunk_backward``: one chunk with carried state under such a mask, with a key bias [B|1, H, Sk]
  or a pair bias [B, H, Sq, Sk] (``chunk_bias``: ALiBi as the kernels see one chunk);
* ``dense_attention`` / ``dense_attention_bwd``: the whole sequence with flash-attn's causal / ``window_size``
  (bottom-right aligned), ALiBi slopes and documents ``cu_seqlens``.

A row that sees no key has O = 0, lse = -inf and no gradient.
"""
from __future__ import annotations

import math

import torch

from oracle import attention_oracle as orc

NEG_INF = float("-inf")


def doc_ids(pos, cu):
    """Document of each position in ``pos`` (the last d with cu[d] <= pos; zero-length documents are skipped)."""
    cu = torch.as_tensor(cu, dtype=torch.int64)
    return torch.searchsorted(cu[:-1], torch.as_tensor(pos, dtype=torch.int64), right=True) - 1


def same_doc(pos_q, pos_k, cu):
    """[len(pos_q), len(pos_k)] bool: the two positions share a document."""
    return doc_ids(pos_q, cu).unsqueeze(1) == doc_ids(pos_k, cu).unsqueeze(0)


def mask_of(sq, sk, mask, device=None):
    """[sq, sk] bool of a kernel mask (see the module docstring) on ``device``, or None when nothing is masked."""
    if mask is None or mask == "none":
        return None
    a = torch.arange(sq, device=device).unsqueeze(1)
    b = torch.arange(sk, device=device).unsqueeze(0)
    if mask[0] == "causal_offset":
        return b <= a + int(mask[1])
    assert mask[0] in ("band", "doc"), mask
    lo, hi = mask[1], mask[2]
    m = torch.ones(sq, sk, dtype=torch.bool, device=device)
    if lo is not None:
        m &= b >= a + int(lo)
    if hi is not None:
        m &= b <= a + int(hi)
    if mask[0] == "doc":
        _, _, _, cu, q_pos0, k_pos0, ps = mask
        m &= same_doc(q_pos0 + ps * torch.arange(sq), k_pos0 + ps * torch.arange(sk), list(cu)).to(device)
    return m


def window_mask(sq, sk, window, causal=False):
    """[sq, sk] bool: key j visible to row i iff i + sk - sq - left <= j <= i + sk - sq + right (-1: that side
    unlimited; ``causal`` forces right = 0), or None when nothing is masked."""
    left, right = (-1, -1) if window is None else (int(window[0]), int(window[1]))
    if causal:
        right = 0
    if left < 0 and right < 0:
        return None
    off = sk - sq
    return mask_of(sq, sk, ("band", None if left < 0 else off - left, None if right < 0 else off + right))


def bias(slopes, pos_q, pos_k):
    """fp64 [B, H, Sq, Sk]: the ALiBi bias -slopes[b, h] |pos_q(a) - pos_k(c)| (slopes [B, H]; int64 positions)."""
    d = (pos_q.view(-1, 1) - pos_k.view(1, -1)).double()
    return -slopes.double().view(*slopes.shape, 1, 1) * d.abs()


def chunk_bias(alibi, sq, sk):
    """The ALiBi bias of one chunk of ``sq`` rows and ``sk`` keys, ``alibi = (slopes [B, H], dist0, pstride)``: row a
    and key c are d = pstride (a - c) + dist0 apart.  On the slopes' device."""
    slopes, dist0, pstride = alibi
    pos = lambda n: pstride * torch.arange(n, dtype=torch.int64, device=slopes.device)  # noqa: E731
    return bias(slopes, pos(sq) + int(dist0), pos(sk))


def std_slopes(H):
    """flash-attn's standard slopes 2^(-8 (h + 1) / H), fp32."""
    return torch.tensor([2.0 ** (-8.0 * (h + 1) / H) for h in range(H)], dtype=torch.float32)


def slopes_for(B, H, per_batch, seed=0):
    """fp32 slopes: ``(H,)`` standard ones, or ``(B, H)`` scaled by a per-(batch, head) factor in [0.5, 1.5)."""
    if not per_batch:
        return std_slopes(H)
    g = torch.Generator().manual_seed(seed)
    return std_slopes(H).view(1, H) * (0.5 + torch.rand(B, H, generator=g))


def as_bh(slopes, B):
    return slopes.view(1, -1).expand(B, -1) if slopes.dim() == 1 else slopes


def _scores(q, k, scale, bias, dtype):
    s = torch.einsum("bqhd,bkhd->bhqk", q.to(dtype), k.to(dtype)) * scale
    if bias is not None:
        s = s + (bias.to(dtype) if bias.dim() == 4 else bias.to(dtype).unsqueeze(2))
    return s


def _softmax(s, m):
    """(p, lse) of masked scores; rows that see nothing: p = 0, lse = -inf."""
    if m is not None:
        s = s.masked_fill(~m, NEG_INF)
    lse = torch.logsumexp(s, dim=-1)
    dead = torch.isinf(lse) & (lse < 0)
    p = torch.exp(s - torch.where(dead, torch.zeros_like(lse), lse).unsqueeze(-1))
    return torch.where(dead.unsqueeze(-1), torch.zeros_like(p), p), lse


def _delegated(mask, bias):
    """The masks and biases ``attention_oracle``'s own chunk functions take."""
    return (mask is None or mask == "none" or mask[0] == "causal_offset") and (bias is None or bias.dim() == 3)


def chunk_forward(q, k, v, o_acc, lse, scale, mask=None, dtype=torch.float64, bias=None):
    """``attention_oracle.chunk_forward`` under any kernel mask (``mask_of``), with a key or pair ``bias``."""
    if _delegated(mask, bias):
        return orc.chunk_forward(q, k, v, o_acc, lse, scale, mask or "none", dtype, bias)
    p, lse_i = _softmax(_scores(q, k, scale, bias, dtype), mask_of(q.shape[1], k.shape[1], mask, q.device))
    o_i = torch.einsum("bhqk,bkhd->bqhd", p, v.to(dtype))
    if o_acc is None:
        return o_i, lse_i
    o_acc, lse = o_acc.to(dtype), lse.to(dtype)
    new_lse = torch.logaddexp(lse, lse_i)
    both_empty = torch.isinf(new_lse) & (new_lse < 0)
    w_old = torch.where(both_empty, torch.zeros_like(lse), torch.exp(lse - new_lse))
    w_new = torch.where(both_empty, torch.zeros_like(lse), torch.exp(lse_i - new_lse))
    return w_old.permute(0, 2, 1).unsqueeze(-1) * o_acc + w_new.permute(0, 2, 1).unsqueeze(-1) * o_i, new_lse


def chunk_backward(do, q, k, v, delta, lse, scale, mask=None, dtype=torch.float64, bias=None):
    """``attention_oracle.chunk_backward`` under any kernel mask (``mask_of``), with a key or pair ``bias``; lse is
    the final lse (+inf or a huge value for rows that saw nothing)."""
    if _delegated(mask, bias):
        return orc.chunk_backward(do, q, k, v, delta, lse, scale, mask or "none", dtype, bias)
    do, q, k, v, delta, lse = (t.to(dtype) for t in (do, q, k, v, delta, lse))
    p = torch.exp(_scores(q, k, scale, bias, dtype) - lse.unsqueeze(-1))
    m = mask_of(q.shape[1], k.shape[1], mask, q.device)
    if m is not None:
        p = p.masked_fill(~m, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv


def _dense_softmax(q, k, scale, causal, window, slopes, cu, dtype):
    """(p, lse) over the whole sequence; positions bottom-right aligned (row i at i + Sk - Sq)."""
    sq, sk = q.shape[1], k.shape[1]
    b = None if slopes is None else bias(slopes, torch.arange(sq, dtype=torch.int64) + sk - sq,
                                         torch.arange(sk, dtype=torch.int64))
    m = window_mask(sq, sk, window, causal)
    if cu is not None:
        d = same_doc(torch.arange(sq), torch.arange(sk), cu)
        m = d if m is None else d & m
    return _softmax(_scores(q, k, scale, b, dtype), m)


def dense_attention(q, k, v, scale=None, causal=False, window=None, slopes=None, cu=None, dtype=torch.float64):
    """softmax(q k^T scale + ALiBi, window, documents) v over the whole sequence: (o [B,Sq,H,D], lse [B,H,Sq]).
    ``slopes`` [B, H] (``as_bh``); K/V at the query heads."""
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    p, lse = _dense_softmax(q, k, scale, causal, window, slopes, cu, dtype)
    return torch.einsum("bhqk,bkhd->bqhd", p, v.to(dtype)), lse


def dense_attention_bwd(q, k, v, do, scale=None, causal=False, window=None, slopes=None, cu=None,
                        dtype=torch.float64):
    """(o, lse, dq, dk, dv) of ``dense_attention``."""
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    q, k, v, do = (t.to(dtype) for t in (q, k, v, do))
    p, lse = _dense_softmax(q, k, scale, causal, window, slopes, cu, dtype)
    o = torch.einsum("bhqk,bkhd->bqhd", p, v)
    delta = (o * do).sum(-1).permute(0, 2, 1)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return o, lse, torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv
