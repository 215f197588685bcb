"""The operator boundary of the ring drivers: the five device operations one ring
round needs.  Mirrors the reference's ``attn_forward`` / ``attn_backward`` dispatch
(burst_attn_interface.py:40-93) but with the carried state folded into the
forward call and fp32 accumulation folded into the backward call.

``NativeOps`` is the only implementation in the product: thin calls into the
C-ABI library.  (Tests inject an oracle-backed implementation of the same five
methods to exercise the ring schedules on CPU/gloo; the product never does.)

All tensors are 4-D with head_dim last and contiguous; ``seq_dim`` says which
axis is the sequence (1: flash layout [B,S,H,D]; 2: normal layout [B,H,S,D]).
lse / delta are fp32 [B,H,S].  K and V (and dK / dV) may have fewer heads than Q
(grouped-query attention: query head h reads K/V head h // (Hq // Hkv)); the number
of K/V heads is taken from ``k``.
"""
from __future__ import annotations

import torch

from . import native as _n


def _dims(t: torch.Tensor, seq_dim: int):
    return t.shape[0], t.shape[seq_dim], t.shape[3 - seq_dim], t.shape[3]


def _mask_args(causal, causal_offset, bias, lower, alibi, doc):
    """The chunk entry point of a call's masks and the arguments that differ between the entry points:
    ``("_band", (key bias,), masks)``, ``("_alibi", (), masks + ALiBi)`` or ``("_doc", (), masks + documents)``, with
    masks = (mask_mode, causal_offset, lower_offset).  The key bias goes after v in the forward, after lse in the
    backward; the mask and variant arguments follow the scale.  A call without ALiBi or documents goes to
    ``ba_*_chunk_band`` with or without a lower edge: with BA_MASK_LOWER clear it is ``ba_*_chunk_gqa``."""
    masks = ((_n.BA_MASK_CAUSAL if causal else _n.BA_MASK_NONE) | (0 if lower is None else _n.BA_MASK_LOWER),
             int(causal_offset), 0 if lower is None else int(lower))
    if doc is not None:
        assert bias is None and alibi is None, "documents are not combined with a key bias or ALiBi"
        cu, n_docs, q_pos0, k_pos0, pstride = doc  # cu_seqlens: int32 device boundaries
        assert cu.dim() == 1 and cu.dtype == torch.int32 and cu.is_contiguous()
        return "_doc", (), masks + (cu.data_ptr(), int(n_docs), int(q_pos0), int(k_pos0), int(pstride))
    if alibi is not None:
        assert bias is None, "ALiBi is not combined with a key bias"
        slopes, dist0, pstride = alibi  # slopes: fp32 [B, H]
        assert slopes.dim() == 2 and slopes.stride(1) == 1 and slopes.dtype == torch.float32
        return "_alibi", (), masks + (slopes.data_ptr(), slopes.stride(0), int(dist0), int(pstride))
    return "_band", (_n.rs(bias),), masks


class NativeOps:
    name = "sm90"
    tile_head_dims = (64, 128)  # head dims the tile kernels are built for; the drivers zero-pad others up

    def __init__(self):
        self.lib = _n.lib()  # raises if the library is missing -- no fallback
        self.launches = 0    # kernels launched through this object (bench.py's gpu_launches)
        self.timing = None   # bench.py: {kernel name: [(start_event, end_event), ...]} when enabled
        self.shapes = {}

    def enable_timing(self, on=True):
        """Bracket every launch with CUDA events on the launching stream (bench.py roofline)."""
        self.timing = {} if on else None
        if on:
            self.shapes = {}  # {kernel name: {(Sq, Sk, H, causal): launches}} since timing was switched on

    def _t0(self, dev):
        if self.timing is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record(torch.cuda.current_stream(dev))
        return e

    def _t1(self, name, e0, dev):
        if e0 is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record(torch.cuda.current_stream(dev))
            self.timing.setdefault(name, []).append((e0, e1))

    def _shape(self, name, Sq, Sk, H, causal):
        if self.timing is not None:
            d = self.shapes.setdefault(name, {})
            key = (int(Sq), int(Sk), int(H), bool(causal))
            d[key] = d.get(key, 0) + 1

    def dominant_shape(self, name):
        """(Sq, Sk, H, causal) of most launches of `name` since enable_timing (bench.py: ncu traffic lookup)."""
        d = self.shapes.get(name)
        return max(d, key=d.get) if d else None

    def kernel_ms(self):
        """{kernel name: (launches, total ms)} -- call after a synchronize."""
        return {k: (len(v), sum(a.elapsed_time(b) for a, b in v)) for k, v in (self.timing or {}).items()}

    # ---- forward round: fold chunk (k, v) into (o_acc, lse); on last write o_out
    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None, alibi=None, doc=None):
        """bias: optional fp32 [B|1, H, Sk] additive bias per key (expanded views with stride 0 over the batch are fine),
        indexed by the query head.  lower: optional lower edge of a band mask, key c visible to row a only if
        c >= a + lower (None: no lower edge).  alibi: optional ``(slopes, dist0, pstride)``, the bias
        -slopes[b, h] |pstride (a - c) + dist0| with slopes fp32 [B, H] (stride 0 over the batch is fine); not
        combined with ``bias``.  doc: optional ``(cu_seqlens, n_docs, q_pos0, k_pos0, pstride)``, packed documents:
        row a (at position q_pos0 + pstride a) sees key c (at k_pos0 + pstride c) only inside one document of the
        int32 device boundaries cu_seqlens; not combined with ``bias`` or ``alibi``."""
        B, Sq, H, D = _dims(q, seq_dim)
        Sk, H_kv = k.shape[seq_dim], k.shape[3 - seq_dim]
        flags = (_n.BA_FWD_FIRST if first else 0) | (_n.BA_FWD_LAST if last else 0)
        e0 = self._t0(q.device)
        entry, bias_arg, masks = _mask_args(causal, causal_offset, bias, lower, alibi, doc)
        rc = getattr(self.lib, "ba_fwd_chunk" + entry)(
            _n.t4(q, seq_dim), _n.t4(k, seq_dim), _n.t4(v, seq_dim), *bias_arg, _n.t4(o_acc, seq_dim), _n.rs(lse),
            _n.t4(o_out, seq_dim), B, Sq, Sk, H, H_kv, D, float(scale), *masks, flags, _n.dtype_code(q.dtype),
            _n.stream_ptr(q.device))
        _n.check(rc, "ba_fwd_chunk")
        self._shape("fwd_chunk_kernel", Sq, Sk, H, causal)
        self._t1("fwd_chunk_kernel", e0, q.device)
        self.launches += 1

    # ---- delta = rowsum(O * dO)
    def delta(self, o, d_o, out, seq_dim):
        B, S, H, D = _dims(o, seq_dim)
        e0 = self._t0(o.device)
        rc = self.lib.ba_bwd_delta(_n.t4(o, seq_dim), _n.t4(d_o, seq_dim), _n.rs(out), B, S, H, D,
                                   _n.dtype_code(o.dtype), _n.stream_ptr(o.device))
        _n.check(rc, "ba_bwd_delta")
        self._t1("delta_kernel", e0, o.device)
        self.launches += 1

    # ---- backward round: accumulate into fp32 dq_acc / dk_acc / dv_acc
    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None, alibi=None, doc=None):
        """lower, alibi, doc: as in fwd_chunk."""
        B, Sq, H, D = _dims(q, seq_dim)
        Sk, H_kv = k.shape[seq_dim], k.shape[3 - seq_dim]
        e0 = self._t0(q.device)
        entry, bias_arg, masks = _mask_args(causal, causal_offset, bias, lower, alibi, doc)
        rc = getattr(self.lib, "ba_bwd_chunk" + entry)(
            _n.t4(d_o, seq_dim), _n.t4(q, seq_dim), _n.t4(k, seq_dim), _n.t4(v, seq_dim), _n.rs(delta), _n.rs(lse),
            *bias_arg, _n.t4(dq_acc, seq_dim), _n.t4(dk_acc, seq_dim), _n.t4(dv_acc, seq_dim), B, Sq, Sk, H, H_kv, D,
            float(scale), *masks, 1 if deterministic else 0, _n.dtype_code(q.dtype), _n.stream_ptr(q.device))
        _n.check(rc, "ba_bwd_chunk")
        self._shape("bwd_chunk_kernel", Sq, Sk, H, causal)
        self._t1("bwd_chunk_kernel", e0, q.device)
        self.launches += 1

    # ---- dst (16-bit) = src (fp32)
    def cast(self, src, dst, seq_dim):
        B, S, H, D = _dims(src, seq_dim)
        e0 = self._t0(src.device)
        rc = self.lib.ba_cast_from_f32(_n.t4(src, seq_dim), _n.t4(dst, seq_dim), B, S, H, D,
                                       _n.dtype_code(dst.dtype), _n.stream_ptr(src.device))
        _n.check(rc, "ba_cast_from_f32")
        self._t1("cast_kernel", e0, src.device)
        self.launches += 1

    # ---- dst (fp32) += src (fp32)
    def accumulate(self, src, dst, seq_dim):
        B, S, H, D = _dims(src, seq_dim)
        e0 = self._t0(src.device)
        rc = self.lib.ba_accumulate_f32(_n.t4(src, seq_dim), _n.t4(dst, seq_dim), B, S, H, D,
                                        _n.stream_ptr(src.device))
        _n.check(rc, "ba_accumulate_f32")
        self._t1("accumulate_kernel", e0, src.device)
        self.launches += 1


_ops = None
_ops_override = None


def get_ops():
    """The chunk operators used by the ring drivers (native; created lazily)."""
    global _ops
    if _ops_override is not None:
        return _ops_override
    if _ops is None:
        _ops = NativeOps()
    return _ops


def _set_ops_for_testing(ops):
    """tests/ only: run the ring schedules against a different set of chunk
    operators (the CPU oracle under gloo).  Pass None to restore the native ops."""
    global _ops_override
    _ops_override = ops
