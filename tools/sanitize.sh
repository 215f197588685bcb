#!/bin/bash
# compute-sanitizer over the tile kernels at small shapes (SURVEY.md 5.2): memcheck (global / shared out-of-bounds),
# racecheck (shared-memory hazards between the warp roles), synccheck (barrier misuse).  1 GPU, a few minutes.
#   bash tools/sanitize.sh > sanitize.txt 2>&1
# The mbarrier/TMA/wgmma async proxies are only partly modelled by the tools: treat racecheck hazards on the
# TMA-written operand tiles as advisory, memcheck / synccheck findings as bugs.
set -x
CASE='import sys; sys.path.insert(0, "burst-attention_b200"); sys.path.insert(0, "tests"); import torch
from burst_attn import burst_attn_func
torch.manual_seed(0)
for D, causal in ((128, False), (128, True), (64, True)):
    q, k, v, do = (torch.randn(1, 384, 2, D, device="cuda", dtype=torch.bfloat16) for _ in range(4))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, "cuda", causal)
    g = torch.autograd.grad(o, (qq, kk, vv), do)
torch.cuda.synchronize(); print("ran")'
for tool in memcheck synccheck racecheck; do
  timeout 600 compute-sanitizer --tool $tool --kernel-regex kns=ba python -c "$CASE" 2>&1 | tail -25
done
