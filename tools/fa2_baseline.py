"""Informational baseline on the same box: the kernels the REFERENCE runs on this path --
flash-attn 2.8.x `_flash_attn_forward/_backward` (FA2, mma.sync SASS; what
burst_utils.py:149-249 calls) -- timed on the bench shapes.  flash_attn is an installed library,
not part of this repo's product path; nothing here is used by bench.py's value."""
import json
import sys

import torch

try:
    from flash_attn import flash_attn_func
except Exception as e:  # noqa: BLE001
    print(json.dumps({"fa2": "unavailable", "why": repr(e)}))
    sys.exit(0)


def t(fn, n=3):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


out = {}
for S in (32768, 65536):
    for causal in (False, True):
        H, D = 32, 128
        q, k, v = (torch.randn(1, S, H, D, device="cuda", dtype=torch.bfloat16, requires_grad=True) for _ in range(3))
        do = torch.randn(1, S, H, D, device="cuda", dtype=torch.bfloat16)
        ms_f = t(lambda: flash_attn_func(q, k, v, causal=causal))
        o = flash_attn_func(q, k, v, causal=causal)
        ms_b = t(lambda: torch.autograd.grad(o, (q, k, v), do, retain_graph=True))
        f = 4.0 * S * S * H * D / (2 if causal else 1)
        out[f"S{S}_causal{int(causal)}"] = {"fwd_ms": ms_f, "fwd_tflops": f / ms_f / 1e9, "bwd_ms": ms_b,
                                            "bwd_tflops": 2.5 * f / ms_b / 1e9,
                                            "fwd_bwd_tflops": 3.5 * f / (ms_f + ms_b) / 1e9}
print(json.dumps({"fa2_flash_attn": out}))
