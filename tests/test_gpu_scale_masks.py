"""Windows, ALiBi and packed documents at the sequence length their benchmarks time (tools/bench_window.py,
bench_alibi.py, bench_varlen.py): S = 65536 through the public API with the default L2 block, so that the 32768 split
runs as in the benchmarks.  Whole heads of O, dQ, dK and dV are held to the 16-bit error model (``lowp_model``) by
the row-blocked oracle and model of ``scale_model``:

* heads 0 and H - 1 (for ALiBi the steepest and the flattest slope) and one seeded head; under GQA whole K/V groups;
* rows that see no key must give O = dQ = 0 and keys no row sees dK = dV = 0, exactly;
* one workload per mask family runs with ``deterministic=True`` twice: the two runs agree bitwise.

The public calls return no lse; the backward, which reads it, is held to the model instead.
``test_report`` prints the worst bound usage per output and the peak device memory.
"""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func  # noqa: E402
from burst_attn.flash_triton import flash_attn_func, flash_attn_varlen_func  # noqa: E402
import lowp_model as lm  # noqa: E402
import mask_oracle as mo  # noqa: E402
import scale_model as sm  # noqa: E402

S, D = 65536, 128
SEAM = 32768  # the forward's default L2 split of 65536 keys: the state is carried across it


def _mix(S):
    """bench_varlen's seeded "mix256-16384" document lengths."""
    rng = random.Random(2024)
    mixed, left = [], S
    while left > 0:
        n = min(left, rng.randint(256, 16384))
        mixed.append(n)
        left -= n
    return mixed


def _cu(lengths):
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    return cu


U2048, MIX, U16 = _cu([2048] * (S // 2048)), _cu(_mix(S)), _cu([16] * (S // 16))

# id: (call, H, Hkv, dtype, window (left, right) or None, causal, alibi, documents, deterministic, row block)
WORK = {
    "win1024": ("flash", 32, 32, torch.bfloat16, (1024, 0), True, False, None, False, 4096),
    "win16384": ("flash", 32, 32, torch.bfloat16, (16384, 0), True, False, None, False, 2048),
    "win2sided": ("burst", 32, 32, torch.bfloat16, (2047, 511), False, False, None, True, 4096),
    "alibi_causal": ("burst", 32, 32, torch.bfloat16, None, True, True, None, True, 1024),
    "alibi_full": ("burst", 32, 32, torch.bfloat16, None, False, True, None, False, 1024),
    "doc2048": ("varlen", 32, 32, torch.bfloat16, None, True, False, U2048, False, 4096),
    "docmix": ("burst", 32, 32, torch.bfloat16, None, True, False, MIX, True, 2048),
    "doc16_gqa": ("varlen", 32, 8, torch.bfloat16, None, True, False, U16, False, 4096),
    "doc_win": ("burst", 32, 32, torch.bfloat16, (300, 0), True, False, U2048, False, 4096),
    "fp16_win": ("flash", 8, 8, torch.float16, (1024, 0), True, False, None, False, 4096),
    "fp16_alibi": ("burst", 8, 8, torch.float16, None, True, True, None, False, 1024),
    "fp16_doc": ("varlen", 8, 8, torch.float16, None, True, False, U2048, False, 4096),
}


def _mask(window, causal, cu):
    """The whole call in the kernels' mask language (rows and keys both 0 .. S - 1)."""
    left, right = (None, None) if window is None else window
    hi = 0 if causal else right
    lo = None if left is None else -left
    if cu is not None:
        return ("doc", lo, hi, tuple(cu), 0, 0, 1)
    if lo is None:
        return None if hi is None else ("causal_offset", hi)
    return ("band", lo, hi)


def _call(kind, q, k, v, window, causal, slopes, cu, det):
    ws = (-1, -1) if window is None else window
    if kind == "flash":
        return flash_attn_func(q, k, v, None, causal, None, ws, slopes)
    if kind == "varlen":
        cut = torch.tensor(cu, dtype=torch.int32, device=q.device)
        n = max(b - a for a, b in zip(cu, cu[1:]))
        return flash_attn_varlen_func(q[0], k[0], v[0], cut, cut, n, n, causal=causal, window_size=ws,
                                      deterministic=det).unsqueeze(0)
    cut = None if cu is None else torch.tensor(cu, dtype=torch.int32, device=q.device)
    return burst_attn_func(q, k, v, None, "cuda", causal, False, det, None, [None, None], ws, slopes, cut)


def _grads(kind, q, k, v, do, window, causal, slopes, cu, det):
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    o = _call(kind, qq, kk, vv, window, causal, slopes, cu, det)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    return o.detach(), dq, dk, dv


def _inputs(H, Hkv, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda h: torch.randn(1, S, h, D, device="cuda", generator=g, dtype=dtype)  # noqa: E731
    return rn(H), rn(Hkv), rn(Hkv), rn(H)


@pytest.mark.parametrize("wid", list(WORK))
def test_whole_heads_at_65536(wid):
    kind, H, Hkv, dtype, window, causal, alibi, cu, det, block = WORK[wid]
    seed = 1234 + list(WORK).index(wid)
    q, k, v, do = _inputs(H, Hkv, dtype, seed)
    slopes = mo.std_slopes(H).cuda() if alibi else None
    out = _grads(kind, q, k, v, do, window, causal, slopes, cu, det)
    if det:
        again = _grads(kind, q, k, v, do, window, causal, slopes, cu, det)
        for n, a, b in zip(("o", "dq", "dk", "dv"), out, again):
            assert torch.equal(a, b), f"{wid}: deterministic {n} differs between two runs"
        del again
    G = H // Hkv
    pick = random.Random(seed).randrange(1, Hkv - 1)  # one seeded K/V group besides the first and the last
    heads = sorted({h for hk in (0, pick, Hkv - 1) for h in range(hk * G, hk * G + G)})
    if G > 1:
        heads = list(range(pick * G, pick * G + G))  # a whole K/V group
    al = None if slopes is None else (slopes.view(1, H), 0, 1)
    sm.check_api(wid, out, q, k, v, do, _mask(window, causal, cu), al, heads, block, seams=(SEAM,))
    del out, q, k, v, do
    torch.cuda.empty_cache()


def test_report():
    """Runs last: the worst error / bound per output and workload, and the peak device memory of this file."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(lm.WORST.items()):
        print(f"worst {name:>4s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
