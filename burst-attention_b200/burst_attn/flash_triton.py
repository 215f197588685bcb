"""Single-GPU attention entry points with the reference's names and signatures
(burst_attn/flash_triton.py:1013-1160: ``flash_attn_func``, ``flash_attn_kvpacked_func``,
``flash_attn_qkvpacked_func``; layout [batch, seqlen, nheads, headdim], ``causal`` bottom-right aligned like the
Triton kernel's ``seqlen_k - seqlen_q`` offset).  The reference keeps a vanilla Triton FlashAttention copy there
that its ring op never calls; here the three wrappers run the same sm_90a tile kernels as the ring (one local
"round", no communication), reading Q / K / V straight out of the packed tensor through strided views (TMA takes
the strides; nothing is unpacked or copied on the way in).

``bias`` (the Triton copy's additive attention bias, lao.py:102-105,155-173): the per-KEY form -- shape
``(batch | 1, nheads, 1, seqlen_k)``, the reference's "vector" bias, e.g. a key-padding mask of -inf (ALiBi has its
own argument, ``alibi_slopes``) -- runs in the tile kernels (forward: one extra K = 16 step on the tensor core per
score tile; backward: a per-thread scalar in the exponent's FMA).  The "matrix" form ``(.., seqlen_q, seqlen_k)`` is
not supported (at the sequence lengths this path is built for it does not fit memory) and raises.  As in the reference no gradient
flows into the bias.

Grouped-query / multi-query attention as in flash-attn: ``flash_attn_func`` and ``flash_attn_kvpacked_func`` accept
K/V with ``nheads_k`` heads where ``nheads_k`` divides ``nheads``; query head ``h`` attends with K/V head
``h // (nheads // nheads_k)``, and dK / dV come back with ``nheads_k`` heads (summed over each group).  A per-key bias
is still ``(batch | 1, nheads, 1, seqlen_k)``, one row per query head.

Sliding-window (local) attention as in flash-attn: ``window_size=(left, right)``, -1 for an unlimited side; query row
``i`` sees key ``j`` iff ``i + Sk - Sq - left <= j <= i + Sk - Sq + right`` (the bottom-right alignment of ``causal``,
which forces ``right = 0``).  The tile kernels skip the key tiles outside each row block's band.  A row that sees no
key returns 0 and gets no gradient.

ALiBi as in flash-attn: ``alibi_slopes``, fp32 ``(nheads,)`` or ``(batch, nheads)`` indexed by the query head, adds
``-slope |i + Sk - Sq - j|`` to the score of query row ``i`` and key ``j`` (bottom-right aligned).  It combines with
``causal``, ``window_size`` and grouped-query attention, not with ``bias``; no gradient flows into the slopes.

Packed documents as in flash-attn 2: ``flash_attn_varlen_func`` takes ``(total, nheads, headdim)`` operands and the
boundaries ``cu_seqlens_q`` / ``cu_seqlens_k`` (which must be equal: self-attention packing), and runs ONE launch plan
over the packed sequence, each row attending only to keys of its own document (with ``causal`` / ``window_size``
inside it) -- instead of one launch chain per document.
"""
from __future__ import annotations

import math

import torch

from .burst_attn_interface import (_band, _BandForward, _bwd_band_launches, _bwd_band_run, _check_alibi,
                                   _check_cu_seqlens, _check_window, _doc_trim, _fwd_band_launches, _pad_head_dim,
                                   _positions, _unpad)
from .chunk_ops import get_ops

__all__ = ["flash_attn_func", "flash_attn_kvpacked_func", "flash_attn_qkvpacked_func", "flash_attn_varlen_func"]


def _key_bias(bias, q, k):
    """(batch | 1, nheads, 1, seqlen_k) -> fp32 [B|1 (stride 0), H, Sk] view for the chunk operators."""
    if bias is None:
        return None
    B, H, Sk = q.shape[0], q.shape[2], k.shape[1]
    if bias.dim() != 4 or bias.shape[2] != 1 or bias.shape[3] != Sk or bias.shape[1] != H or bias.shape[0] not in (1, B):
        raise NotImplementedError(f"only a per-key bias of shape (batch | 1, {H}, 1, {Sk}) is supported by the sm_90a "
                                  f"tile kernels, got {tuple(bias.shape)}")
    b3 = bias.detach().to(torch.float32).reshape(bias.shape[0], H, Sk).contiguous()
    return b3.expand(B, H, Sk)


def _local_pieces(band, Sq, Sk, docs=None):
    """The one piece (``_round_pieces`` form) of a local call, bottom-right aligned, or none when no row sees a key;
    with documents (Sq == Sk) trimmed to the rows and keys that share one."""
    left, right = band
    off = Sk - Sq
    b = _band(Sq, Sk, None if left is None else off - left, None if right is None else off + right)
    pieces = [] if b is None else [(0, Sq, 0, Sk) + b]
    if docs is not None:
        pos, _ = _positions("local", 1, 0, Sq)
        pieces = [p for p in (_doc_trim(p, docs[0], pos, pos, 1) for p in pieces) if p is not None]
    return pieces


def _local_doc(docs, Sq):
    """The documents of a local call (``_ring_doc`` form: positions are the row and key indices), or None."""
    if docs is None:
        return None
    pos, _ = _positions("local", 1, 0, Sq)
    return docs[1], len(docs[0]) - 1, pos, pos, 1


def _local_alibi(slopes, Sq, Sk):
    """The ALiBi of a local call (bottom-right aligned: row i sits at position i + Sk - Sq), or None."""
    if slopes is None:
        return None
    pos_q, _ = _positions("local", 1, Sk - Sq, Sq)
    pos_k, _ = _positions("local", 1, 0, Sk)
    return slopes, pos_q, pos_k, 1


def _local_forward(q, k, v, softmax_scale, bias, band, alibi, docs=None):
    ops = get_ops()
    scale = softmax_scale or 1.0 / math.sqrt(q.shape[-1])
    (qp, kp, vp), D = _pad_head_dim(ops, [q, k, v])
    B, Sq, H = qp.shape[0], qp.shape[1], qp.shape[2]
    out = torch.empty(qp.shape, dtype=qp.dtype, device=qp.device)
    lse = torch.empty((B, H, Sq), dtype=torch.float32, device=qp.device)
    launches = _fwd_band_launches(_local_pieces(band, Sq, kp.shape[1], docs))
    state = _BandForward([launches], qp, lse, Sq)
    state.run(ops, launches, qp, kp, vp, lse, out, scale, 1, bias, _local_alibi(alibi, Sq, kp.shape[1]),
              _local_doc(docs, Sq))
    state.finish(ops, out, 1)
    return out, lse, scale, (qp, kp, vp), D


def _local_backward(do, qp, kp, vp, out, lse, scale, bias, band, alibi, deterministic=False, docs=None):
    ops = get_ops()
    (g,), _ = _pad_head_dim(ops, [do])
    g, out = g.contiguous(), out.contiguous()
    B, Sq, H = qp.shape[0], qp.shape[1], qp.shape[2]
    delta = torch.empty((B, H, Sq), dtype=torch.float32, device=qp.device)
    ops.delta(out, g, delta, 1)
    f32 = dict(dtype=torch.float32, device=qp.device)
    dq, dk, dv = torch.zeros(qp.shape, **f32), torch.zeros(kp.shape, **f32), torch.zeros(vp.shape, **f32)
    _bwd_band_run(ops, _bwd_band_launches(_local_pieces(band, Sq, kp.shape[1], docs)), g, qp, kp, vp, delta, lse, dq,
                  dk, dv, scale, 1, deterministic, bias, _local_alibi(alibi, Sq, kp.shape[1]), _local_doc(docs, Sq))
    return dq, dk, dv


def _cast(src, like, D):
    dst = torch.empty(src.shape, dtype=like.dtype, device=src.device)
    get_ops().cast(src, dst, 1)
    return _unpad(dst, D)


def _check(bias, *ts):
    for t in ts:
        assert t.stride(-1) == 1, "the head_dim axis must be contiguous"


def _alibi(alibi_slopes, bias, q):
    slopes = _check_alibi(alibi_slopes, q, 2)
    if slopes is not None and bias is not None:
        raise NotImplementedError("alibi_slopes together with a per-key bias is not supported")
    return slopes


def _check_heads(q, k):
    hq, hkv = q.shape[2], k.shape[2]
    assert hkv > 0 and hq % hkv == 0, f"nheads ({hq}) must be a multiple of nheads_k ({hkv})"


class FlashAttnFunc(torch.autograd.Function):
    """q: (batch, seqlen_q, nheads, headdim); k, v: (batch, seqlen_k, nheads_k, headdim), nheads_k | nheads
    (reference :1122-1168)."""

    @staticmethod
    def forward(ctx, q, k, v, bias=None, causal=False, softmax_scale=None, window_size=(-1, -1), alibi_slopes=None):
        _check(bias, q, k, v)
        _check_heads(q, k)
        ctx.bias = _key_bias(bias, q, k)
        ctx.band = _check_window(window_size, causal)
        ctx.alibi = _alibi(alibi_slopes, bias, q)
        out, lse, ctx.softmax_scale, saved, ctx.head_dim = _local_forward(q, k, v, softmax_scale, ctx.bias, ctx.band,
                                                                          ctx.alibi)
        ctx.save_for_backward(*saved, out, lse)
        return _unpad(out, ctx.head_dim)

    @staticmethod
    def backward(ctx, do):
        qp, kp, vp, out, lse = ctx.saved_tensors
        dq, dk, dv = _local_backward(do, qp, kp, vp, out, lse, ctx.softmax_scale, ctx.bias, ctx.band, ctx.alibi)
        return (_cast(dq, qp, ctx.head_dim), _cast(dk, kp, ctx.head_dim), _cast(dv, vp, ctx.head_dim), None, None, None,
                None, None)


class FlashAttnKVPackedFunc(torch.autograd.Function):
    """q: (batch, seqlen_q, nheads, headdim); kv: (batch, seqlen_k, 2, nheads_k, headdim), nheads_k | nheads
    (reference :1073-1119)."""

    @staticmethod
    def forward(ctx, q, kv, bias=None, causal=False, softmax_scale=None, window_size=(-1, -1), alibi_slopes=None):
        _check(bias, q, kv)
        _check_heads(q, kv[:, :, 0])
        ctx.bias = _key_bias(bias, q, kv[:, :, 0])
        ctx.band = _check_window(window_size, causal)
        ctx.alibi = _alibi(alibi_slopes, bias, q)
        out, lse, ctx.softmax_scale, saved, ctx.head_dim = _local_forward(q, kv[:, :, 0], kv[:, :, 1],
                                                                          softmax_scale, ctx.bias, ctx.band, ctx.alibi)
        ctx.save_for_backward(*saved, out, lse)
        return _unpad(out, ctx.head_dim)

    @staticmethod
    def backward(ctx, do):
        qp, kp, vp, out, lse = ctx.saved_tensors
        dq, dk, dv = _local_backward(do, qp, kp, vp, out, lse, ctx.softmax_scale, ctx.bias, ctx.band, ctx.alibi)
        dkv = torch.stack([_cast(dk, kp, ctx.head_dim), _cast(dv, vp, ctx.head_dim)], dim=2)
        return _cast(dq, qp, ctx.head_dim), dkv, None, None, None, None, None


class FlashAttnQKVPackedFunc(torch.autograd.Function):
    """qkv: (batch, seqlen, 3, nheads, headdim)  (reference :1021-1070)."""

    @staticmethod
    def forward(ctx, qkv, bias=None, causal=False, softmax_scale=None, window_size=(-1, -1), alibi_slopes=None):
        _check(bias, qkv)
        ctx.bias = _key_bias(bias, qkv[:, :, 0], qkv[:, :, 1])
        ctx.band = _check_window(window_size, causal)
        ctx.alibi = _alibi(alibi_slopes, bias, qkv[:, :, 0])
        out, lse, ctx.softmax_scale, saved, ctx.head_dim = _local_forward(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2],
                                                                          softmax_scale, ctx.bias, ctx.band, ctx.alibi)
        ctx.save_for_backward(*saved, out, lse)
        return _unpad(out, ctx.head_dim)

    @staticmethod
    def backward(ctx, do):
        qp, kp, vp, out, lse = ctx.saved_tensors
        dq, dk, dv = _local_backward(do, qp, kp, vp, out, lse, ctx.softmax_scale, ctx.bias, ctx.band, ctx.alibi)
        dqkv = torch.stack([_cast(t, qp, ctx.head_dim) for t in (dq, dk, dv)], dim=2)
        return dqkv, None, None, None, None, None


class FlashAttnVarlenFunc(torch.autograd.Function):
    """q: (total, nheads, headdim); k, v: (total, nheads_k, headdim), nheads_k | nheads; documents cu_seqlens
    (flash-attn 2's ``flash_attn_varlen_func``, self-attention packing)."""

    @staticmethod
    def forward(ctx, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p, softmax_scale, causal,
                window_size, softcap, alibi_slopes, deterministic, return_attn_probs):
        if dropout_p != 0.0:
            raise NotImplementedError("flash_attn_varlen_func: dropout_p != 0 is not supported")
        if softcap != 0.0:
            raise NotImplementedError("flash_attn_varlen_func: softcap != 0 is not supported")
        if alibi_slopes is not None:
            raise NotImplementedError("flash_attn_varlen_func: alibi_slopes is not supported with documents")
        if return_attn_probs:
            raise NotImplementedError("flash_attn_varlen_func: return_attn_probs is not supported")
        if q.dim() != 3 or k.dim() != 3 or k.shape != v.shape or q.shape[0] != k.shape[0] or q.shape[2] != k.shape[2]:
            raise ValueError("flash_attn_varlen_func: q must be (total, nheads, headdim) and k, v (total, nheads_k, "
                             f"headdim) with the same total, got {tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
        docs = _check_cu_seqlens(cu_seqlens_q, q.shape[0], q.device, "cu_seqlens_q")
        docs_k = _check_cu_seqlens(cu_seqlens_k, k.shape[0], q.device, "cu_seqlens_k")
        if docs[0] != docs_k[0]:
            raise NotImplementedError("flash_attn_varlen_func: cu_seqlens_q must equal cu_seqlens_k (self-attention "
                                      "packing); cross-attention packing is not supported")
        longest = max(b - a for a, b in zip(docs[0], docs[0][1:]))
        for name, m in (("max_seqlen_q", max_seqlen_q), ("max_seqlen_k", max_seqlen_k)):
            if int(m) < longest:
                raise ValueError(f"flash_attn_varlen_func: {name} = {m} is below the longest document ({longest})")
        q4, k4, v4 = q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0)  # one packed sequence of batch 1
        _check(None, q4, k4, v4)
        _check_heads(q4, k4)
        ctx.band = _check_window(window_size, causal)
        ctx.docs, ctx.deterministic = docs, deterministic
        out, lse, ctx.softmax_scale, saved, ctx.head_dim = _local_forward(q4, k4, v4, softmax_scale, None, ctx.band,
                                                                          None, docs)
        ctx.save_for_backward(*saved, out, lse)
        return _unpad(out, ctx.head_dim)[0]

    @staticmethod
    def backward(ctx, do):
        qp, kp, vp, out, lse = ctx.saved_tensors
        dq, dk, dv = _local_backward(do.unsqueeze(0), qp, kp, vp, out, lse, ctx.softmax_scale, None, ctx.band, None,
                                     ctx.deterministic, ctx.docs)
        return (_cast(dq, qp, ctx.head_dim)[0], _cast(dk, kp, ctx.head_dim)[0], _cast(dv, vp, ctx.head_dim)[0]) + \
            (None,) * 12


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0,
                           softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0, alibi_slopes=None,
                           deterministic=False, return_attn_probs=False):
    """flash-attn 2's varlen entry point for packed self-attention: q (total, nheads, headdim), k and v (total,
    nheads_k, headdim); document d holds rows cu_seqlens_q[d] .. cu_seqlens_q[d + 1] - 1 (int32, equal for q and k).
    ``causal`` and ``window_size`` apply inside each document.  Raises NotImplementedError for unequal boundaries,
    dropout, softcap, alibi_slopes and return_attn_probs."""
    return FlashAttnVarlenFunc.apply(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p,
                                     softmax_scale, causal, window_size, softcap, alibi_slopes, deterministic,
                                     return_attn_probs)


flash_attn_func = FlashAttnFunc.apply
flash_attn_kvpacked_func = FlashAttnKVPackedFunc.apply
flash_attn_qkvpacked_func = FlashAttnQKVPackedFunc.apply
