"""Packed documents (cu_seqlens): fwd+bwd time and TFLOP/s over the visible (query, key) pairs, per document mix.

    python tools/bench_varlen.py [--seq 65536] [--steps 10] [--warmup 3] [--mixes uniform2048,...] [--hkv 32]

Workload: bf16, d = 128, bs = 1, H = 32, W = 1, causal, S = 65536 packed as uniform 2048-token documents, uniform 8192,
and a seeded mix of 256 .. 16384 (--mixes also offers uniform16: 4096 documents; --hkv < 32: grouped-query K/V).  For
each mix it times, alternating step by step after warm-up:
  varlen     flash_attn_varlen_func over the packed (S, H, d) sequence
  burst      burst_attn_func(cu_seqlens=...) on the [1, S, H, d] sequence
  loop       flash_attn_func once per document (the workaround without documents; not run above 1024 documents)
  causal     burst_attn_func over the whole sequence, no documents (what the packing would cost unmasked)
Each step (forward + backward) is timed with CUDA events.  FLOPs count the visible pairs of the documents (causal
inside each one) for the first three and of the whole causal sequence for the last: 4 d per pair and head forward,
10 d backward.  Prints one JSON line per (mix, method), then the card name, power limit and SM clock read in the same
process.  Writes nothing.
"""
import argparse
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench_window import _device_info  # noqa: E402
from burst_attn import burst_attn_func  # noqa: E402
from burst_attn.flash_triton import flash_attn_func, flash_attn_varlen_func  # noqa: E402

H, D = 32, 128


def mixes(S):
    rng = random.Random(2024)
    mixed, left = [], S
    while left > 0:
        n = min(left, rng.randint(256, 16384))
        mixed.append(n)
        left -= n
    return {"uniform2048": [2048] * (S // 2048), "uniform8192": [8192] * (S // 8192), "mix256-16384": mixed,
            "uniform16": [16] * (S // 16)}


def _grad(fn, q, k, v, do):
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    return torch.autograd.grad(fn(qq, kk, vv), (qq, kk, vv), do)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mixes", default="uniform2048,uniform8192,mix256-16384")
    ap.add_argument("--hkv", type=int, default=H, help="K/V heads (grouped-query attention when < 32)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_varlen.py measures on the GPU; there is no CPU path"
    dev = torch.device("cuda", 0)
    S = args.seq
    g = torch.Generator(device=dev).manual_seed(1234)
    q, do = (torch.randn(1, S, H, D, device=dev, generator=g, dtype=torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(1, S, args.hkv, D, device=dev, generator=g, dtype=torch.bfloat16) for _ in range(2))
    results = []
    for name in args.mixes.split(","):
        lens = mixes(S)[name]
        cu_list = [0]
        for n in lens:
            cu_list.append(cu_list[-1] + n)
        cu = torch.tensor(cu_list, dtype=torch.int32, device=dev)
        longest = max(lens)
        methods = {
            "varlen": lambda a, b, c: flash_attn_varlen_func(a[0], b[0], c[0], cu, cu, longest, longest,
                                                             causal=True)[None],
            "burst": lambda a, b, c: burst_attn_func(a, b, c, None, "cuda", True, False, False, None, [None, None],
                                                     (-1, -1), None, cu),
            "loop": lambda a, b, c: torch.cat([flash_attn_func(a[:, s:e], b[:, s:e], c[:, s:e], None, True)
                                               for s, e in zip(cu_list, cu_list[1:]) if e > s], 1),
            "causal": lambda a, b, c: burst_attn_func(a, b, c, None, "cuda", True),
        }
        if len(lens) > 1024:
            del methods["loop"]
        times = {m: [] for m in methods}
        for i in range(args.warmup + args.steps):
            for m, fn in methods.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _grad(fn, q, k, v, do)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[m].append(e0.elapsed_time(e1))
        doc_pairs = sum(n * (n + 1) // 2 for n in lens)
        for m in methods:
            pairs = S * (S + 1) // 2 if m == "causal" else doc_pairs
            ms = statistics.median(times[m])
            results.append({"seq": S, "mix": name, "n_docs": len(lens), "hkv": args.hkv, "method": m,
                            "visible_pairs": pairs,
                            "ms_per_step": round(ms, 3), "ms_min": round(min(times[m]), 3),
                            "tflops_visible": round(14 * D * H * pairs / (ms * 1e-3) / 1e12, 1)})
    info = _device_info(dev)
    for r in results:
        print(json.dumps(r), flush=True)
    print(json.dumps({"device": info, "torch": torch.__version__}), flush=True)


if __name__ == "__main__":
    main()
