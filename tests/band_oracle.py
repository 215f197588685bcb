"""fp64 CPU oracle of sliding-window (band) attention, for the tests only.

``oracle/attention_oracle.py`` states the reference's masks (none / causal / causal offset); this module adds the band
the window tests need, in the same conventions (flash layout [B, S, H, D], math in fp64):

* ``window_mask``: flash-attn's ``window_size=(left, right)`` with its bottom-right alignment;
* ``dense_attention`` / ``dense_attention_bwd``: the whole sequence under a window;
* ``band_mask`` and ``chunk_forward`` / ``chunk_backward``: one chunk with carried state under the kernels' band mask
  ``("band", lo, hi)`` -- key b visible to row a iff a + lo <= b <= a + hi, None for an open side -- restating
  ``attention_oracle.chunk_forward`` / ``chunk_backward`` with that mask.

A row that sees no key has O = 0, lse = -inf and no gradient.
"""
from __future__ import annotations

import math

import torch

from oracle import attention_oracle as orc

NEG_INF = float("-inf")


def window_mask(sq, sk, window, causal=False):
    """[sq, sk] bool: key j visible to row i iff i + sk - sq - left <= j <= i + sk - sq + right (-1: that side
    unlimited; ``causal`` forces right = 0), or None when nothing is masked."""
    left, right = (-1, -1) if window is None else (int(window[0]), int(window[1]))
    if causal:
        right = 0
    if left < 0 and right < 0:
        return None
    off = sk - sq
    return band_mask(sq, sk, ("band", None if left < 0 else off - left, None if right < 0 else off + right))


def band_mask(sq, sk, mask):
    """[sq, sk] bool of a kernel mask: None, ("causal_offset", off) or ("band", lo, hi)."""
    if mask is None or mask == "none":
        return None
    a = torch.arange(sq).unsqueeze(1)
    b = torch.arange(sk).unsqueeze(0)
    if mask[0] == "causal_offset":
        return b <= a + int(mask[1])
    assert mask[0] == "band", mask
    _, lo, hi = mask
    m = torch.ones(sq, sk, dtype=torch.bool)
    if lo is not None:
        m &= b >= a + int(lo)
    if hi is not None:
        m &= b <= a + int(hi)
    return m


def _scores(q, k, scale, key_bias, dtype):
    s = torch.einsum("bqhd,bkhd->bhqk", q.to(dtype), k.to(dtype)) * scale
    if key_bias is not None:
        s = s + key_bias.to(dtype).unsqueeze(2)
    return s


def _softmax(s, m):
    """(p, lse) of masked scores; rows that see nothing: p = 0, lse = -inf."""
    if m is not None:
        s = s.masked_fill(~m, NEG_INF)
    lse = torch.logsumexp(s, dim=-1)
    dead = torch.isinf(lse) & (lse < 0)
    p = torch.exp(s - torch.where(dead, torch.zeros_like(lse), lse).unsqueeze(-1))
    return torch.where(dead.unsqueeze(-1), torch.zeros_like(p), p), lse


def dense_attention(q, k, v, scale=None, causal=False, window=None, dtype=torch.float64):
    """softmax(q k^T scale, window) v over the whole sequence: (o [B,Sq,H,D], lse [B,H,Sq])."""
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    s = _scores(q, k, scale, None, dtype)
    p, lse = _softmax(s, window_mask(q.shape[1], k.shape[1], window, causal))
    return torch.einsum("bhqk,bkhd->bqhd", p, v.to(dtype)), lse


def dense_attention_bwd(q, k, v, do, scale=None, causal=False, window=None, dtype=torch.float64):
    """(o, lse, dq, dk, dv) of ``dense_attention``."""
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    q, k, v, do = (t.to(dtype) for t in (q, k, v, do))
    p, lse = _softmax(_scores(q, k, scale, None, dtype), window_mask(q.shape[1], k.shape[1], window, causal))
    o = torch.einsum("bhqk,bkhd->bqhd", p, v)
    delta = (o * do).sum(-1).permute(0, 2, 1)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return o, lse, torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv


def chunk_forward(q, k, v, o_acc, lse, scale, mask=None, dtype=torch.float64, key_bias=None):
    """``attention_oracle.chunk_forward`` under a kernel mask (``band_mask``)."""
    if mask is None or mask == "none" or mask[0] != "band":
        return orc.chunk_forward(q, k, v, o_acc, lse, scale, mask or "none", dtype, key_bias)
    p, lse_i = _softmax(_scores(q, k, scale, key_bias, dtype), band_mask(q.shape[1], k.shape[1], mask))
    o_i = torch.einsum("bhqk,bkhd->bqhd", p, v.to(dtype))
    if o_acc is None:
        return o_i, lse_i
    o_acc, lse = o_acc.to(dtype), lse.to(dtype)
    new_lse = torch.logaddexp(lse, lse_i)
    both_empty = torch.isinf(new_lse) & (new_lse < 0)
    w_old = torch.where(both_empty, torch.zeros_like(lse), torch.exp(lse - new_lse))
    w_new = torch.where(both_empty, torch.zeros_like(lse), torch.exp(lse_i - new_lse))
    return w_old.permute(0, 2, 1).unsqueeze(-1) * o_acc + w_new.permute(0, 2, 1).unsqueeze(-1) * o_i, new_lse


def chunk_backward(do, q, k, v, delta, lse, scale, mask=None, dtype=torch.float64, key_bias=None):
    """``attention_oracle.chunk_backward`` under a kernel mask (``band_mask``); lse is the final lse (+inf or a huge
    value for rows that saw nothing)."""
    if mask is None or mask == "none" or mask[0] != "band":
        return orc.chunk_backward(do, q, k, v, delta, lse, scale, mask or "none", dtype, key_bias)
    do, q, k, v, delta, lse = (t.to(dtype) for t in (do, q, k, v, delta, lse))
    p = torch.exp(_scores(q, k, scale, key_bias, dtype) - lse.unsqueeze(-1))
    p = p.masked_fill(~band_mask(q.shape[1], k.shape[1], mask), 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv
