"""fp64 CPU oracle of ALiBi attention, for the tests only.

Row a and key c get the bias ``-slopes[b, h] |d|``, d the distance of the pair: over a whole sequence of positions
``d = pos_q(a) - pos_k(c)``; in one chunk, as the kernels see it, ``d = pstride (a - c) + dist0``.  The functions
restate ``band_oracle`` (flash layout [B, S, H, D], fp64) with that bias:

* ``dense_attention_bwd``: the whole sequence, with flash-attn's causal / window_size (bottom-right aligned);
* ``chunk_forward`` / ``chunk_backward``: one chunk with carried state under the kernels' masks (None,
  ("causal_offset", off) or ("band", lo, hi)) and ``alibi = (slopes [B, H], dist0, pstride)``.

A row that sees no key has O = 0, lse = -inf and no gradient.
"""
from __future__ import annotations

import torch

import band_oracle as bo


def bias(slopes, pos_q, pos_k):
    """fp64 [B, H, Sq, Sk]: -slopes[b, h] |pos_q(a) - pos_k(c)| (slopes [B, H]; positions int64 vectors)."""
    d = (pos_q.view(-1, 1) - pos_k.view(1, -1)).double()
    return -slopes.double().view(*slopes.shape, 1, 1) * d.abs()


def chunk_bias(alibi, sq, sk):
    """The bias of one chunk of ``sq`` rows and ``sk`` keys: d = pstride (a - c) + dist0."""
    slopes, dist0, pstride = alibi
    return bias(slopes, pstride * torch.arange(sq, dtype=torch.int64) + int(dist0),
                pstride * torch.arange(sk, dtype=torch.int64))


def _softmax(s, m):
    return bo._softmax(s, m)


def dense_attention_bwd(q, k, v, do, scale, causal, window, slopes):
    """(o, lse, dq, dk, dv) over the whole sequence (k / v at the query heads); positions bottom-right aligned."""
    q, k, v, do = (t.double() for t in (q, k, v, do))
    sq, sk = q.shape[1], k.shape[1]
    b = bias(slopes, torch.arange(sq, dtype=torch.int64) + sk - sq, torch.arange(sk, dtype=torch.int64))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale + b
    p, lse = _softmax(s, bo.window_mask(sq, sk, window, causal))
    o = torch.einsum("bhqk,bkhd->bqhd", p, v)
    delta = (o * do).sum(-1).permute(0, 2, 1)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return o, lse, torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv


def chunk_forward(q, k, v, o_acc, lse, scale, mask, alibi):
    """``band_oracle.chunk_forward`` with the chunk's ALiBi."""
    q, k, v = (t.double() for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale + chunk_bias(alibi, q.shape[1], k.shape[1])
    p, lse_i = _softmax(s, bo.band_mask(q.shape[1], k.shape[1], mask))
    o_i = torch.einsum("bhqk,bkhd->bqhd", p, v)
    if o_acc is None:
        return o_i, lse_i
    o_acc, lse = o_acc.double(), lse.double()
    new_lse = torch.logaddexp(lse, lse_i)
    empty = torch.isinf(new_lse) & (new_lse < 0)
    w_old = torch.where(empty, torch.zeros_like(lse), torch.exp(lse - new_lse))
    w_new = torch.where(empty, torch.zeros_like(lse), torch.exp(lse_i - new_lse))
    return w_old.permute(0, 2, 1).unsqueeze(-1) * o_acc + w_new.permute(0, 2, 1).unsqueeze(-1) * o_i, new_lse


def chunk_backward(do, q, k, v, delta, lse, scale, mask, alibi):
    """``band_oracle.chunk_backward`` with the chunk's ALiBi; lse is the final lse (+inf or huge for dead rows)."""
    do, q, k, v, delta, lse = (t.double() for t in (do, q, k, v, delta, lse))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale + chunk_bias(alibi, q.shape[1], k.shape[1])
    p = torch.exp(s - lse.unsqueeze(-1))
    m = bo.band_mask(q.shape[1], k.shape[1], mask)
    if m is not None:
        p = p.masked_fill(~m, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv


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

