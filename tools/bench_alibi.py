"""ALiBi: fwd+bwd time per step with and without ``alibi_slopes``, causal and non-causal.

    python tools/bench_alibi.py [--seq 65536] [--steps 10] [--warmup 3]

Workload: bf16, d = 128, bs = 1, H = 32, flash-attn's standard slopes 2^(-8 (h + 1) / H).  Two calls are timed:
flash_attn_func and burst_attn_func at W = 1 (one rank, no process group), each on the whole sequence.  Each step
(forward + backward) is timed with CUDA events; the variants with and without ALiBi alternate step by step after
warm-up, so clock drift hits both alike.  Prints one JSON line per (call, causal) with the median ms per step of
each and their ratio, then the card name, power limit and SM clock read in the same process.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench_window import _device_info  # noqa: E402
from burst_attn import burst_attn_func  # noqa: E402
from burst_attn.flash_triton import flash_attn_func  # noqa: E402

H, D = 32, 128


def _step(call, q, k, v, do, causal, slopes):
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    if call == "burst_attn_func":
        o = burst_attn_func(qq, kk, vv, None, "cuda", causal, False, False, None, [None, None], (-1, -1), slopes)
    else:
        o = flash_attn_func(qq, kk, vv, None, causal, None, (-1, -1), slopes)
    return torch.autograd.grad(o, (qq, kk, vv), do)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_alibi.py measures on the GPU; there is no CPU path"
    dev = torch.device("cuda", 0)
    S = args.seq
    g = torch.Generator(device=dev).manual_seed(1234)
    q, k, v, do = (torch.randn(1, S, H, D, device=dev, generator=g, dtype=torch.bfloat16) for _ in range(4))
    slopes = torch.tensor([2.0 ** (-8.0 * (h + 1) / H) for h in range(H)], dtype=torch.float32, device=dev)
    for call in ("flash_attn_func", "burst_attn_func"):
        for causal in (True, False):
            times = {False: [], True: []}
            for i in range(args.warmup + args.steps):
                for alibi in (False, True):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    _step(call, q, k, v, do, causal, slopes if alibi else None)
                    e1.record()
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        times[alibi].append(e0.elapsed_time(e1))
            base, ali = statistics.median(times[False]), statistics.median(times[True])
            print(json.dumps({"call": call, "seq": S, "causal": causal, "ms_per_step": round(base, 3),
                              "ms_per_step_alibi": round(ali, 3), "ratio": round(ali / base, 4),
                              "ms_min": round(min(times[False]), 3), "ms_min_alibi": round(min(times[True]), 3),
                              **_device_info(dev)}), flush=True)
    print(json.dumps({"device": _device_info(dev), "torch": torch.__version__}), flush=True)


if __name__ == "__main__":
    main()
