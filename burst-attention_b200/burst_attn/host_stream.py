"""Host-resident operands (single rank): ``burst_attn_func`` called with CPU tensors in pinned memory.

The L2-blocked drivers (burst_attn_interface.py ``_fwd_round`` / ``_bwd_round``) consume K/V block by block in the
forward and finish dQ row block by row block in the backward, so when Q/K/V/dO live in HOST memory the copies can
ride under the kernels instead of bracketing the call:

  forward   up   : Q, then K/V block c on the upload stream (event per block); the kernel of block c waits for it
            down : O after the last block -- under the backward, if one follows
  backward  up   : dO row block r (event per block); delta and the backward kernel of block r wait for it
            down : dQ row block r as soon as its sub-launch has finished; the LAST row block is launched per key
                   block so that dK / dV blocks finish -- and leave -- progressively instead of all at the end

Exposed at S = 262144 (H = 32, d = 128): Q + the first K/V block up (2.6 GB) and the last dQ / dK / dV blocks down
(0.8 GB) out of 17 GB each way.  Device memory: the 16-bit Q, K, V, O stay resident between forward and backward.

Contract (the same as ``tensor.to("cpu", non_blocking=True)``): the returned host tensors are complete after
``torch.cuda.synchronize()``; the compute stream itself is made to wait for every copy at the end of the backward.
Only W = 1 (no ring); with W > 1 pass device tensors.
"""
from __future__ import annotations

import torch

from .burst_attn_interface import _bwd_rows, _fwd_blocks
from .chunk_ops import get_ops

_streams = {}


def _copy_streams(dev):
    key = dev.index
    if key not in _streams:
        _streams[key] = (torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev))
    return _streams[key]


def _blocks(S, blk):
    return [(c0, min(blk, S - c0)) for c0 in range(0, S, blk)]


def _pinned_like(shape, dtype):
    return torch.empty(shape, dtype=dtype, pin_memory=True)


def is_host_call(q, k, v) -> bool:
    return q.device.type == "cpu" and k.device.type == "cpu" and v.device.type == "cpu" and torch.cuda.is_available()


def forward(q, k, v, scale, seq_dim, causal, blk):
    """q, k, v: pinned CPU [B,S,H,D] (seq_dim 1) or [B,H,S,D] (seq_dim 2).  Returns (o_host, saved device tensors)."""
    ops = get_ops()
    dev = torch.device("cuda", torch.cuda.current_device())
    cur = torch.cuda.current_stream(dev)
    up, down = _copy_streams(dev)
    for t in (q, k, v):
        assert t.is_pinned(), "host-resident operands must be in pinned memory (tensor.pin_memory())"
    B, S, H = q.shape[0], q.shape[seq_dim], q.shape[3 - seq_dim]
    Sk = k.shape[seq_dim]
    qd, kd, vd = (torch.empty(t.shape, dtype=t.dtype, device=dev) for t in (q, k, v))
    out = torch.empty_like(qd)
    lse = torch.empty((B, H, S), dtype=torch.float32, device=dev)
    kblocks = _blocks(Sk, blk)
    n = len(kblocks)
    o_acc = torch.empty(qd.shape, dtype=torch.float32, device=dev) if (n > 1 or causal) else None
    up.wait_stream(cur)  # the fresh device buffers may reuse memory the compute stream is still working on
    ev = []
    with torch.cuda.stream(up):
        qd.copy_(q, non_blocking=True)
        for c0, cn in kblocks:
            kd.narrow(seq_dim, c0, cn).copy_(k.narrow(seq_dim, c0, cn), non_blocking=True)
            vd.narrow(seq_dim, c0, cn).copy_(v.narrow(seq_dim, c0, cn), non_blocking=True)
            e = torch.cuda.Event()
            e.record(up)
            ev.append(e)
    for t in (qd, kd, vd):
        t.record_stream(up)
    _fwd_blocks(ops, qd, kd, vd, o_acc, lse, out, scale, causal, 0, True, True, seq_dim, blk,
                before=lambda c: cur.wait_event(ev[c]))
    o_host = _pinned_like(q.shape, q.dtype)
    done = torch.cuda.Event()
    done.record(cur)
    with torch.cuda.stream(down):
        down.wait_event(done)
        o_host.copy_(out, non_blocking=True)
    out.record_stream(down)
    return o_host, (qd, kd, vd, out, lse)


def backward(d_o, saved, scale, seq_dim, causal, blk, deterministic):
    """d_o: pinned CPU gradient of O.  Returns pinned CPU (dq, dk, dv)."""
    ops = get_ops()
    qd, kd, vd, out, lse = saved
    dev = qd.device
    cur = torch.cuda.current_stream(dev)
    up, down = _copy_streams(dev)
    if not d_o.is_pinned():
        d_o = d_o.pin_memory()
    d_o = d_o.contiguous()
    B, S, H = qd.shape[0], qd.shape[seq_dim], qd.shape[3 - seq_dim]
    Sk = kd.shape[seq_dim]
    f32 = dict(dtype=torch.float32, device=dev)
    g = torch.empty(qd.shape, dtype=qd.dtype, device=dev)
    delta = torch.empty((B, H, S), **f32)
    dq_acc, dk_acc, dv_acc = torch.zeros(qd.shape, **f32), torch.zeros(kd.shape, **f32), torch.zeros(vd.shape, **f32)
    dq16, dk16, dv16 = torch.empty_like(qd), torch.empty_like(kd), torch.empty_like(vd)
    dq_h, dk_h, dv_h = (_pinned_like(t.shape, t.dtype) for t in (qd, kd, vd))
    rblocks, kblocks = _blocks(S, blk), _blocks(Sk, blk)
    up.wait_stream(cur)
    ev = []
    with torch.cuda.stream(up):
        for r0, rn in rblocks:
            g.narrow(seq_dim, r0, rn).copy_(d_o.narrow(seq_dim, r0, rn), non_blocking=True)
            e = torch.cuda.Event()
            e.record(up)
            ev.append(e)
    g.record_stream(up)
    down.wait_stream(cur)

    def ship(acc, lowp, host, s0, sn):
        """fp32 accumulator rows [s0, s0+sn) -> 16 bit on the compute stream -> host on the download stream."""
        ops.cast(acc.narrow(seq_dim, s0, sn), lowp.narrow(seq_dim, s0, sn), seq_dim)
        e = torch.cuda.Event()
        e.record(cur)
        with torch.cuda.stream(down):
            down.wait_event(e)
            host.narrow(seq_dim, s0, sn).copy_(lowp.narrow(seq_dim, s0, sn), non_blocking=True)

    for i, (r0, rn) in enumerate(rblocks):
        cur.wait_event(ev[i])
        gb, qb = g.narrow(seq_dim, r0, rn), qd.narrow(seq_dim, r0, rn)
        db, lb = delta.narrow(2, r0, rn), lse.narrow(2, r0, rn)
        ops.delta(out.narrow(seq_dim, r0, rn), gb, db, seq_dim)
        dqb = dq_acc.narrow(seq_dim, r0, rn)
        if i < len(rblocks) - 1:
            _bwd_rows(ops, g, qd, kd, vd, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, 0, seq_dim, deterministic,
                      r0, rn)
            ship(dq_acc, dq16, dq_h, r0, rn)
            continue
        # last row block: one launch per key block, so every dK / dV block is final right after its launch
        for k0, kn in kblocks:
            if not causal or k0 <= r0 + rn - 1:
                ops.bwd_chunk(gb, qb, kd.narrow(seq_dim, k0, kn), vd.narrow(seq_dim, k0, kn), db, lb, dqb,
                              dk_acc.narrow(seq_dim, k0, kn), dv_acc.narrow(seq_dim, k0, kn), scale, causal,
                              r0 - k0, seq_dim, deterministic)
            ship(dk_acc, dk16, dk_h, k0, kn)
            ship(dv_acc, dv16, dv_h, k0, kn)
        ship(dq_acc, dq16, dq_h, r0, rn)
    for t in (dq16, dk16, dv16):
        t.record_stream(down)
    cur.wait_stream(down)  # stream order: whatever follows on the compute stream sees complete host gradients
    return dq_h, dk_h, dv_h
