#!/usr/bin/env python
"""Launch ONE tile kernel at a given launch shape a few times (for a profiler run on one kernel).
  python tools/launch_one.py --kernel bwd --Sq 32768 --Sk 32768 [--H 32] [--causal] [--off 0] [--n 3] [--time]
Inputs are N(0,1) bf16; lse/delta come from a real forward of the same shape when it is cheap, else plausible
constants (timing and traffic do not depend on them)."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "burst-attention_b200"))
import torch  # noqa: E402

from burst_attn.chunk_ops import NativeOps  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--kernel", choices=["fwd", "bwd"], required=True)
ap.add_argument("--Sq", type=int, required=True)
ap.add_argument("--Sk", type=int, required=True)
ap.add_argument("--H", type=int, default=32)
ap.add_argument("--D", type=int, default=128)
ap.add_argument("--causal", action="store_true")
ap.add_argument("--off", type=int, default=0)
ap.add_argument("--n", type=int, default=3)
ap.add_argument("--time", action="store_true")
ap.add_argument("--deterministic", action="store_true")
ap.add_argument("--fresh", action="store_true", help="fwd: first+last in one launch (no carried state, 16-bit output)")
a = ap.parse_args()
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
mk = lambda S: torch.randn(1, S, a.H, a.D, device=dev, generator=g, dtype=torch.float32).to(torch.bfloat16)  # noqa: E731
q, do, k, v = mk(a.Sq), mk(a.Sq), mk(a.Sk), mk(a.Sk)
ops = NativeOps()
scale = a.D ** -0.5
lse = torch.empty(1, a.H, a.Sq, device=dev, dtype=torch.float32)
o_acc = torch.empty(1, a.Sq, a.H, a.D, device=dev, dtype=torch.float32)
out = torch.empty_like(q)
ops.fwd_chunk(q, k, v, o_acc, lse, out, scale, a.causal, a.off, True, True, 1)  # warm-up + real lse
torch.cuda.synchronize()
flops = 4.0 * a.Sq * a.Sk * a.H * a.D / (2.0 if a.causal else 1.0)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
if a.kernel == "fwd":
    e0.record()
    for i in range(a.n):
        ops.fwd_chunk(q, k, v, o_acc, lse, out, scale, a.causal, a.off, a.fresh, a.fresh, 1)  # default: carried-state form
    e1.record()
else:
    delta = torch.empty(1, a.H, a.Sq, device=dev, dtype=torch.float32)
    ops.delta(out, do, delta, 1)
    dq, dk, dv = (torch.zeros(t.shape, device=dev, dtype=torch.float32) for t in (q, k, v))
    ops.bwd_chunk(do, q, k, v, delta, lse, dq, dk, dv, scale, a.causal, a.off, 1, a.deterministic)
    torch.cuda.synchronize()
    flops *= 2.5
    e0.record()
    for i in range(a.n):
        ops.bwd_chunk(do, q, k, v, delta, lse, dq, dk, dv, scale, a.causal, a.off, 1, a.deterministic)
    e1.record()
torch.cuda.synchronize()
if a.time:
    ms = e0.elapsed_time(e1) / a.n
    print(f"{a.kernel} Sq={a.Sq} Sk={a.Sk} H={a.H} D={a.D} causal={a.causal}: {ms:.3f} ms/launch, "
          f"{flops / ms / 1e9:.1f} TFLOP/s")
