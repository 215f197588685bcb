"""fp64 CPU oracle of packed-document attention (flash-attn's ``cu_seqlens``), for the tests only.

A query at position a sees a key at position c iff both lie in one document ``[cu[d], cu[d + 1])`` and c is inside the
causal / window band of a (``band_oracle.window_mask``).  Positions count the full sequence; a shard or a launch gives
its rows and keys as position vectors.  A row that sees no key has O = 0, lse = -inf and no gradient.
"""
from __future__ import annotations

import math

import torch

import band_oracle as bo


def doc_ids(pos, cu):
    """Document of each position in ``pos`` (the last d with cu[d] <= pos; zero-length documents are skipped)."""
    cu = torch.as_tensor(cu, dtype=torch.int64)
    return torch.searchsorted(cu[:-1], torch.as_tensor(pos, dtype=torch.int64), right=True) - 1


def same_doc(pos_q, pos_k, cu):
    """[len(pos_q), len(pos_k)] bool: the two positions share a document."""
    return doc_ids(pos_q, cu).unsqueeze(1) == doc_ids(pos_k, cu).unsqueeze(0)


def visible(S, cu, causal=False, window=None):
    """[S, S] bool over the full sequence: the document mask on top of causal / window."""
    m = same_doc(torch.arange(S), torch.arange(S), cu)
    w = bo.window_mask(S, S, window, causal)
    return m if w is None else m & w


def masked_chunk_forward(q, k, v, o_acc, lse, scale, m, dtype=torch.float64):
    """One chunk under the bool mask m [Sq, Sk], folded into the carried (o_acc, lse) (None: no state)."""
    p, lse_i = bo._softmax(bo._scores(q, k, scale, None, dtype), m)
    o_i = torch.einsum("bhqk,bkhd->bqhd", p, v.to(dtype))
    if o_acc is None:
        return o_i, lse_i
    o_acc, lse = o_acc.to(dtype), lse.to(dtype)
    new_lse = torch.logaddexp(lse, lse_i)
    empty = torch.isinf(new_lse) & (new_lse < 0)
    w_old = torch.where(empty, torch.zeros_like(lse), torch.exp(lse - new_lse))
    w_new = torch.where(empty, torch.zeros_like(lse), torch.exp(lse_i - new_lse))
    return w_old.permute(0, 2, 1).unsqueeze(-1) * o_acc + w_new.permute(0, 2, 1).unsqueeze(-1) * o_i, new_lse


def masked_chunk_backward(do, q, k, v, delta, lse, scale, m, dtype=torch.float64):
    """(dq, dk, dv) of one chunk under the bool mask m; lse is the final lse (huge for rows that saw nothing)."""
    do, q, k, v, delta, lse = (t.to(dtype) for t in (do, q, k, v, delta, lse))
    p = torch.exp(bo._scores(q, k, scale, None, dtype) - lse.unsqueeze(-1)).masked_fill(~m, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    ds = p * (torch.einsum("bqhd,bkhd->bhqk", do, v) - delta.unsqueeze(-1)) * scale
    return torch.einsum("bhqk,bkhd->bqhd", ds, k), torch.einsum("bhqk,bqhd->bkhd", ds, q), dv


def dense_attention_bwd(q, k, v, do, cu, scale=None, causal=False, window=None, dtype=torch.float64):
    """(o, lse, dq, dk, dv) over the whole packed sequence [B, S, H, D] (K/V heads already expanded)."""
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    q, k, v, do = (t.to(dtype) for t in (q, k, v, do))
    m = visible(q.shape[1], cu, causal, window)
    o, lse = masked_chunk_forward(q, k, v, None, None, scale, m, dtype)
    delta = (o * do).sum(-1).permute(0, 2, 1)
    ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
    dq, dk, dv = masked_chunk_backward(do, q, k, v, delta, ls, scale, m, dtype)
    return o, lse, dq, dk, dv
