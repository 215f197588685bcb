"""CPU oracle for the burst-attention hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import this module.  The product
package (``burst-attention_b200/``) never does: it fails loudly when the CUDA
library is missing.

This is a restatement (not a copy) of the reference's algorithm in plain
torch-on-CPU tensor arithmetic, each function citing the reference lines it
follows (paths relative to the reference checkout).  It is pinned against the
reference itself by ``tests/golden/make_golden.py`` (reference imported in the
build container with a ``bmtrain`` stub) -> ``tests/golden/*.npz`` and checked
by ``tests/test_oracle_golden.py``.

Conventions: everything is in the "flash" layout ``[B, S, H, D]`` unless stated;
math is carried out in ``dtype`` (default float64).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch

NEG_INF = float("-inf")


# --------------------------------------------------------------------------- #
# dense reference (what the reference's own test compares against:
# test/test_burst.py:175,184 runs flash_attn_func on the full sequence)
# --------------------------------------------------------------------------- #
def dense_attention(q, k, v, scale=None, causal=False, dtype=torch.float64, bias=None):
    """softmax(q k^T * scale [+ bias] [+ causal mask]) v on the full sequence.

    q,k,v: [B,S,H,D].  bias: optional additive bias broadcastable to [B,H,Sq,Sk], added after the scale exactly
    as the reference's LAO tile does (``qk = qk * softmax_scale + bias``, lao.py:155-173).
    Returns (o [B,S,H,D], lse [B,H,S]) in ``dtype``.
    """
    q, k, v = (t.to(dtype) for t in (q, k, v))
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if bias is not None:
        s = s + bias.to(dtype)
    if causal:
        sq, sk = s.shape[-2:]
        mask = torch.ones(sq, sk, dtype=torch.bool).tril(diagonal=sk - sq)
        s = s.masked_fill(~mask, NEG_INF)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse.unsqueeze(-1))
    o = torch.einsum("bhqk,bkhd->bqhd", p, v)
    return o, lse


def dense_attention_bwd(q, k, v, do, scale=None, causal=False, dtype=torch.float64, bias=None):
    """Analytic gradients of dense_attention (same math autograd would do)."""
    q, k, v, do = (t.to(dtype) for t in (q, k, v, do))
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    o, lse = dense_attention(q, k, v, scale, causal, dtype, bias)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if bias is not None:
        s = s + bias.to(dtype)
    p = torch.exp(s - lse.unsqueeze(-1))
    if causal:
        sq, sk = s.shape[-2:]
        mask = torch.ones(sq, sk, dtype=torch.bool).tril(diagonal=sk - sq)
        p = p.masked_fill(~mask, 0.0)
    delta = (o * do).sum(-1).permute(0, 2, 1)  # [B,H,S]
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    dp = torch.einsum("bqhd,bkhd->bhqk", do, v)
    ds = p * (dp - delta.unsqueeze(-1)) * scale
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, k)
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q)
    return o, lse, dq, dk, dv


# --------------------------------------------------------------------------- #
# per-chunk operator with carried state
# --------------------------------------------------------------------------- #
def _mask(sq: int, sk: int, mask_mode: str, device=None) -> Optional[torch.Tensor]:
    """Visibility mask [sq, sk] for the three kernel mask modes (SURVEY App. B).

    "none": all visible; "causal": key b visible to row a iff b <= a + (sk - sq)
    (bottom-right aligned, what flash-attn's causal flag means and the only way
    the reference calls it: burst_utils.py:150-160); "causal_strict": b < a
    (the reference gets this by slicing q[:,1:] x k[:,:-1] with the causal flag,
    burst_attn_interface.py:463-475).
    """
    if mask_mode == "none":
        return None
    a = torch.arange(sq, device=device).unsqueeze(1)
    b = torch.arange(sk, device=device).unsqueeze(0)
    if isinstance(mask_mode, tuple) and mask_mode[0] == "causal_offset":
        # the kernels' general form: key b visible to row a iff b <= a + offset (views of a larger
        # causal problem: offset = row_start + off - key_start)
        return b <= a + int(mask_mode[1])
    if mask_mode == "causal":
        return b <= a + (sk - sq)
    if mask_mode == "causal_strict":
        return b < a + (sk - sq)
    raise ValueError(mask_mode)


def chunk_forward(q, k, v, o_acc, lse, scale, mask_mode="none", dtype=torch.float64, key_bias=None):
    """One ring round of the forward: attend q to one K/V chunk and merge into
    the running, already-normalised ``(o_acc fp, lse)`` state.

    Follows inter_flash_cuda_fwd (burst_utils.py:149-177): chunk attention ->
    (o_i, lse_i); first round adopts it (:161-163); later rounds merge with
    cuda_scale_out_lse_helper (:20-33):
        new_lse = lse + log(1 + exp(lse_i - lse))
        o = exp(lse - new_lse) * o + exp(lse_i - new_lse) * o_i
    Rows that see no key in this chunk (possible only in "causal_strict") keep
    their state unchanged; the reference reaches the same result by merging only
    the o[:,1:] slice (burst_utils.py:171-174).

    q: [B,Sq,H,D]; k,v: [B,Sk,H,D]; o_acc: [B,Sq,H,D] or None; lse: [B,H,Sq] or None.
    Returns (o_acc, lse).
    """
    q, k, v = (t.to(dtype) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if key_bias is not None:  # [B|1,H,Sk] additive bias per key (the LAO tile's "vector" bias, lao.py:155-173)
        s = s + key_bias.to(dtype).unsqueeze(2)
    m = _mask(s.shape[-2], s.shape[-1], mask_mode, s.device)
    if m is not None:
        s = s.masked_fill(~m, NEG_INF)
    lse_i = torch.logsumexp(s, dim=-1)  # [B,H,Sq]; -inf where nothing visible
    safe = torch.where(torch.isinf(lse_i), torch.zeros_like(lse_i), lse_i)
    p = torch.exp(s - safe.unsqueeze(-1))
    p = torch.where(torch.isinf(lse_i).unsqueeze(-1), torch.zeros_like(p), p)
    o_i = torch.einsum("bhqk,bkhd->bqhd", p, v)
    if o_acc is None:
        return o_i, lse_i
    o_acc, lse = o_acc.to(dtype), lse.to(dtype)
    new_lse = torch.logaddexp(lse, lse_i)
    w_old = torch.exp(lse - new_lse)
    w_new = torch.exp(lse_i - new_lse)
    both_empty = torch.isinf(new_lse) & (new_lse < 0)
    w_old = torch.where(both_empty, torch.zeros_like(w_old), w_old)
    w_new = torch.where(both_empty, torch.zeros_like(w_new), w_new)
    o = w_old.permute(0, 2, 1).unsqueeze(-1) * o_acc + w_new.permute(0, 2, 1).unsqueeze(-1) * o_i
    return o, new_lse


def compute_delta(o, do, dtype=torch.float64):
    """delta = rowsum(O * dO) -> [B,H,S] (burst_attn_interface.py:272-278)."""
    return (o.to(dtype) * do.to(dtype)).sum(-1).permute(0, 2, 1).contiguous()


def chunk_backward(do, q, k, v, delta, lse, scale, mask_mode="none", dtype=torch.float64, key_bias=None):
    """One ring round of the backward for one (Q-bundle, K/V) pair.

    Follows inter_normal_attn_backward (burst_utils.py:77-100), the reference's
    own statement of the chunk math the flash kernel performs:
        p = exp(qk*scale - lse); dv = p^T do; dp = do v^T;
        ds = p * (dp - delta) * scale; dq = ds k; dk = ds^T q
    do,q: [B,Sq,H,D]; k,v: [B,Sk,H,D]; delta,lse: [B,H,Sq] (final, global lse).
    Returns (dq, dk, dv) partials for this pair.
    """
    do, q, k, v, delta, lse = (t.to(dtype) for t in (do, q, k, v, delta, lse))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if key_bias is not None:
        s = s + key_bias.to(dtype).unsqueeze(2)
    p = torch.exp(s - lse.unsqueeze(-1))
    m = _mask(s.shape[-2], s.shape[-1], mask_mode, s.device)
    if m is not None:
        p = p.masked_fill(~m, 0.0)
    dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    dp = torch.einsum("bqhd,bkhd->bhqk", do, v)
    ds = p * (dp - delta.unsqueeze(-1)) * scale
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, k)
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q)
    return dq, dk, dv


# --------------------------------------------------------------------------- #
# reference's "normal"-path chunk state (acc_o un-normalised, m, lse) -- used
# only to pin this oracle against the reference's own CPU-runnable functions.
# --------------------------------------------------------------------------- #
def chunk_forward_unnormalised(q, k, v, m_i, lse_i, acc_o, scale):
    """Restates inter_normal_attn (burst_utils.py:42-74) in [B,H,S,D] layout,
    *including* its +1e-5 inside the log (:71,73) so that golden vectors from
    the reference match to round-off.  Not used by any parity test of the
    product (which uses the exact log)."""
    qk = q @ k.transpose(-2, -1) * scale
    m_ij = qk.max(dim=-1, keepdim=True)[0]
    if m_i is not None:
        m_ij = torch.maximum(m_ij, m_i)
    p = torch.exp(qk - m_ij)
    l_ij = p.sum(dim=-1, keepdim=True)
    pv = (p @ v).to(torch.float32)
    if acc_o is not None:
        acc_o = pv + torch.exp(m_i - m_ij) * acc_o
    else:
        acc_o = pv
    if lse_i is None:
        lse_i = torch.log(l_ij + 1e-5) + m_ij
    else:
        lse_i = torch.log(torch.exp(lse_i - m_ij) + l_ij + 1e-5) + m_ij
    return acc_o, m_ij, lse_i


# --------------------------------------------------------------------------- #
# shard layouts (test/test_burst.py:44-58 get_chunk)
# --------------------------------------------------------------------------- #
def shard(t: torch.Tensor, rank: int, world: int, layout: str, dim: int = 1) -> torch.Tensor:
    """layout: "contiguous" | "zigzag" | "striped"."""
    if layout == "contiguous":
        return t.chunk(world, dim=dim)[rank].contiguous()
    if layout == "zigzag":  # half_reputation: chunks rank and 2W-1-rank
        parts = t.chunk(2 * world, dim=dim)
        return torch.cat([parts[rank], parts[2 * world - 1 - rank]], dim=dim).contiguous()
    if layout == "striped":  # tokens == rank (mod W)
        idx = torch.arange(rank, t.shape[dim], world)
        return t.index_select(dim, idx).contiguous()
    raise ValueError(layout)


def unshard(parts: Sequence[torch.Tensor], layout: str, dim: int = 1) -> torch.Tensor:
    world = len(parts)
    if layout == "contiguous":
        return torch.cat(list(parts), dim=dim)
    if layout == "zigzag":
        halves = [None] * (2 * world)
        for r, p in enumerate(parts):
            a, b = p.chunk(2, dim=dim)
            halves[r], halves[2 * world - 1 - r] = a, b
        return torch.cat(halves, dim=dim)
    if layout == "striped":
        n = sum(p.shape[dim] for p in parts)
        shape = list(parts[0].shape)
        shape[dim] = n
        out = torch.empty(shape, dtype=parts[0].dtype)
        for r, p in enumerate(parts):
            idx = torch.arange(r, n, world)
            out.index_copy_(dim, idx, p)
        return out
    raise ValueError(layout)


# --------------------------------------------------------------------------- #
# single-process ring-schedule simulators (burst_attn_interface.py:214-242 fwd,
# :291-396 bwd; zigzag :209-235,:284-390; striped :454-475,:529-605)
# --------------------------------------------------------------------------- #
def _half(t, idx, dim=1):
    n = t.shape[dim] // 2
    return t.narrow(dim, 0, n) if idx == 0 else t.narrow(dim, n, t.shape[dim] - n)


def ring_forward(qs, ks, vs, scale, mode="none", dtype=torch.float64):
    """Simulate W ranks.  qs/ks/vs: per-rank shards [B,S_loc,H,D].
    mode: "none" (non-causal, contiguous shards), "zigzag" (causal, OpBurstAttn)
    or "striped" (causal, OpBurstAttnStrip).  Returns (o_list, lse_list)."""
    W = len(qs)
    outs, lses = [], []
    for i in range(W):
        o_acc, lse = None, None
        q = qs[i]
        for r in range(1, W + 1):
            j = (i - (r - 1)) % W  # source rank of the held K/V (App. B)
            k, v = ks[j], vs[j]
            if mode == "none":
                o_acc, lse = chunk_forward(q, k, v, o_acc, lse, scale, "none", dtype)
            elif mode == "zigzag":
                if r == 1:
                    o_acc, lse = chunk_forward(q, k, v, o_acc, lse, scale, "causal", dtype)
                elif j < i:  # split_kv (:216,:225-231): all Q x first half of K/V
                    o_acc, lse = chunk_forward(q, _half(k, 0), _half(v, 0), o_acc, lse, scale, "none", dtype)
                else:  # second half of Q x all K/V, merge into o[:, S/2:] (:232-235)
                    n = q.shape[1] // 2
                    o1, l1 = chunk_forward(_half(q, 1), k, v, o_acc[:, n:], lse[:, :, n:], scale, "none", dtype)
                    o_acc = torch.cat([o_acc[:, :n], o1], dim=1)
                    lse = torch.cat([lse[:, :, :n], l1], dim=2)
            elif mode == "striped":
                mm = "causal_strict" if j > i else "causal"  # causal_shift (:454)
                o_acc, lse = chunk_forward(q, k, v, o_acc, lse, scale, mm, dtype)
            else:
                raise ValueError(mode)
        outs.append(o_acc)
        lses.append(lse)
    return outs, lses


def ring_backward(qs, ks, vs, os_, lses, dos, scale, mode="none", dtype=torch.float64):
    """Simulate the backward schedule: K/V stay home on rank i, the Q-bundle
    (delta, dO, Q, lse) of rank j = (i-(r-1)) mod W visits in round r; the dQ
    partial for bundle j accumulates as it travels (one hop behind the bundle)
    and is delivered home to rank j after the final hop (:393-396).
    Returns (dq_list, dk_list, dv_list)."""
    W = len(qs)
    deltas = [compute_delta(os_[i], dos[i], dtype) for i in range(W)]
    dqs = [torch.zeros_like(qs[i], dtype=dtype) for i in range(W)]
    dks = [torch.zeros_like(ks[i], dtype=dtype) for i in range(W)]
    dvs = [torch.zeros_like(vs[i], dtype=dtype) for i in range(W)]
    for r in range(1, W + 1):
        for i in range(W):
            j = (i - (r - 1)) % W
            k, v = ks[i], vs[i]
            q, do, dl, ls = qs[j], dos[j], deltas[j], lses[j]
            if mode == "none":
                dq, dk, dv = chunk_backward(do, q, k, v, dl, ls, scale, "none", dtype)
                dqs[j] += dq; dks[i] += dk; dvs[i] += dv
            elif mode == "zigzag":
                n = q.shape[1] // 2
                if r == 1:
                    dq, dk, dv = chunk_backward(do, q, k, v, dl, ls, scale, "causal", dtype)
                    dqs[j] += dq; dks[i] += dk; dvs[i] += dv
                elif j < i:  # split_q (:294,:322-345): 2nd half of bundle x all K/V
                    dq, dk, dv = chunk_backward(_half(do, 1), _half(q, 1), k, v,
                                                dl[:, :, n:], ls[:, :, n:], scale, "none", dtype)
                    dqs[j][:, n:] += dq; dks[i] += dk; dvs[i] += dv
                else:  # all of bundle x first half of K/V (:347-367,:387-390)
                    dq, dk, dv = chunk_backward(do, q, _half(k, 0), _half(v, 0), dl, ls, scale, "none", dtype)
                    dqs[j] += dq; dks[i][:, :n] += dk; dvs[i][:, :n] += dv
            elif mode == "striped":
                # K home i, Q from j: strict iff j < i and r != 1 (:529)
                mm = "causal_strict" if (j < i and r != 1) else "causal"
                dq, dk, dv = chunk_backward(do, q, k, v, dl, ls, scale, mm, dtype)
                dqs[j] += dq; dks[i] += dk; dvs[i] += dv
            else:
                raise ValueError(mode)
    return dqs, dks, dvs


def get_partition_id_single(r: int) -> int:
    """burst_attn_interface.py:28-29: single ring -> offset r-1."""
    return r - 1


def get_partition_id_double(r: int, intra_rank: int, inter_rank: int, L: int, M: int) -> int:
    """burst_attn_interface.py:27-36 for a double ring of L-rank nodes x M nodes."""
    return ((inter_rank - ((r - 1) // L)) % M) * L + (intra_rank - (r - 1) % L + L) % L


def attention_flops(B, S, H, D, causal=False, mode="fwd") -> float:
    """benchmarks/benchmark.py:17-20."""
    f = 4 * B * S * S * H * D // (2 if causal else 1)
    return {"fwd": f, "bwd": 2.5 * f, "fwd_bwd": 3.5 * f}[mode]
