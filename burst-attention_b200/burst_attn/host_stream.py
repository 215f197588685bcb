"""Host-resident operands (single rank): ``burst_attn_func`` called with CPU tensors in pinned memory.

The launch planner (burst_attn_interface.py) splits a call over L2 blocks: K/V block by block in the forward
(``_fwd_block``) and dQ row block by row block in the backward (``_bwd_block``), so when Q/K/V/dO live in HOST memory
the copies can ride under the kernels instead of bracketing the call:

  forward   up   : Q, then K/V block c on the upload stream (event per block); the kernel of block c waits for it
                   (the forward always splits at the block; first / last duties as in ``_BandForward``)
            down : O after the last block -- under the backward, if one follows
  backward  up   : dO row block r (event per block); delta and the backward kernel of block r wait for it
            down : dQ row block r as soon as its sub-launch has finished; the LAST row block is launched per key
                   block so that dK / dV blocks finish -- and leave -- progressively instead of all at the end

Exposed at S = 262144 (H = 32, d = 128): Q + the first K/V block up (2.6 GB) and the last dQ / dK / dV blocks down
(0.8 GB) out of 17 GB each way.  Device memory: the 16-bit Q, K, V, O stay resident between forward and backward.

Contract: the forward's O is returned like ``tensor.to("cpu", non_blocking=True)``: it rides down under the backward
and is complete after ``torch.cuda.synchronize()``.  The backward's dQ / dK / dV are complete when it returns: the host
waits for their last blocks to land, because autograd hands them to CPU consumers at once (``q.grad += dq`` when
gradients accumulate, tensor hooks, CPU ops upstream of q); the compute stream is made to wait for every copy as well.
Only W = 1 (no ring); with W > 1 pass device tensors.
"""
from __future__ import annotations

import torch

from .burst_attn_interface import _BandForward, _bwd_band_run, _bwd_block, _fwd_block, _round_pieces, _sub
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


def forward(q, k, v, scale, seq_dim, band, blk):
    """q, k, v: pinned CPU [B,S,H,D] (seq_dim 1) or [B,H,S,D] (seq_dim 2); band: the call's (left, right) without a
    window.  Returns (o_host, saved device tensors)."""
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
    piece, = _round_pieces("contiguous", 1, 0, 0, S, Sk, band)
    launches = [x for x in (_fwd_block(piece, c0, cn) for c0, cn in kblocks) if x]
    state = _BandForward([launches], qd, lse, S)
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
    for x in launches:
        cur.wait_event(ev[(x[2] + x[3] - 1) // blk])  # the last K/V block the launch reads
        state.run(ops, [x], qd, kd, vd, lse, out, scale, seq_dim)
    state.finish(ops, out, seq_dim)
    o_host = _pinned_like(q.shape, q.dtype)
    done = torch.cuda.Event()
    done.record(cur)
    with torch.cuda.stream(down):
        down.wait_event(done)
        o_host.copy_(out, non_blocking=True)
    out.record_stream(down)
    return o_host, (qd, kd, vd, out, lse)


def backward(d_o, saved, scale, seq_dim, band, blk, deterministic):
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
    piece, = _round_pieces("contiguous", 1, 0, 0, S, Sk, band)
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

    def run(launch):
        if launch is not None:
            _bwd_band_run(ops, [launch], g, qd, kd, vd, delta, lse, dq_acc, dk_acc, dv_acc, scale, seq_dim,
                          deterministic)

    for i, (r0, rn) in enumerate(rblocks):
        cur.wait_event(ev[i])
        ops.delta(out.narrow(seq_dim, r0, rn), g.narrow(seq_dim, r0, rn), delta.narrow(2, r0, rn), seq_dim)
        if i < len(rblocks) - 1:
            run(_bwd_block(piece, r0, rn))
            ship(dq_acc, dq16, dq_h, r0, rn)
            continue
        # last row block: one launch per key block, so every dK / dV block is final right after its launch
        for k0, kn in kblocks:
            run(_sub(piece, r0, rn, k0, kn))
            ship(dk_acc, dk16, dk_h, k0, kn)
            ship(dv_acc, dv16, dv_h, k0, kn)
        ship(dq_acc, dq16, dq_h, r0, rn)
    for t in (dq16, dk16, dv16):
        t.record_stream(down)
    # autograd hands the gradients to CPU consumers as soon as this returns (AccumulateGrad's q.grad += dq, tensor
    # hooks, CPU ops upstream of q): the host waits for the last blocks to land
    landed = torch.cuda.Event()
    landed.record(down)
    landed.synchronize()
    cur.wait_stream(down)  # stream order: whatever follows on the compute stream sees complete host gradients
    return dq_h, dk_h, dv_h
