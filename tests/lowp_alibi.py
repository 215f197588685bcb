"""The ALiBi edge sweep of the 16-bit model and comparator of ``tests/lowp_model.py``.

``lowp_model.lowp_alibi_forward`` / ``lowp_alibi_backward`` restate what ``fwd_alibi_kernel`` and ``bwd_alibi_kernel``
compute; ``lowp_model.lowp_chain`` / ``oracle_chain`` run them (and the fp64 oracle with each chunk's pair bias) when
given ``alibis``.  lse is held to ``scores_absmax`` in the kernel's frame (``absmax_prefix``: ``|q| |k| scale + slope
(|d| - dref)``), where a chunk millions of positions away adds only a few ulps.

``ALIBI_MUTANTS`` are realistic single faults of the ALiBi arithmetic for the comparator's own tests
(``tests/test_lowp_alibi.py``, ``tests/test_gpu_alibi_edges.py``); ``ALIBI_SWEEP`` is the edge sweep both run;
``tile_classes`` names the sign edges a case's tiles reach.
"""
from __future__ import annotations

import torch

import lowp_model as lm
import mask_oracle as mo

# One realistic fault each.  "_fwd" / "_bwd": only that kernel has the fault.
ALIBI_MUTANTS = (
    "sign_dmin_fwd",         # forward: a tile with dmin in [-pstride, -1] is taken as d >= 0 throughout
    "sign_dmax_fwd",         # forward: a tile with dmax in [1, pstride] is taken as d <= 0 throughout
    "sign_dmin_bwd",         # backward (alibi_tile_sign): the same for dmin
    "sign_dmax_bwd",         # backward (alibi_tile_sign): the same for dmax
    "key_term_no_pstride",   # forward: the per-key term of a one-sign tile is s slope j, without pstride
    "bwd_gqa_first_head",    # backward consumer uses the slope of the group's first query head (the loader does not)
    "carried_not_lowered",   # forward: the carried state's reference is not lowered (alibi_carried_ref skipped)
    "dist0_plus1_fwd",       # forward uses dist0 + 1
    "dist0_plus1_bwd",       # backward uses dist0 + 1
)


def frame_bias(alibi, sq, sk):
    """fp64 [B,H,Sq,Sk]: the bias in the kernel's frame, -slope (|d| - dref) (the chunk's own dref)."""
    slopes, dist0, ps = alibi
    x = lm.distances(sq, sk, dist0, ps).abs() - lm.alibi_dref(sq, sk, dist0, ps).view(-1, 1)
    return -slopes.detach().cpu().double().view(*slopes.shape, 1, 1) * x.double()


def absmax_prefix(q, ks, scale, masks, alibis):
    """``lowp_model.scores_absmax`` over chunks 0..c for every c, in the kernel's frame."""
    sq = q.shape[1]
    fb = [frame_bias(a, sq, k.shape[1]) for a, k in zip(alibis, ks)]
    return [lm.scores_absmax(q, ks[:c + 1], scale, masks[:c + 1], fb[:c + 1]) for c in range(len(ks))]


# --------------------------------------------------------------------------- #
# the ALiBi edge sweep (tests/test_gpu_alibi_edges.py on the kernels, tests/test_lowp_alibi.py on the model)
# --------------------------------------------------------------------------- #
# A case: Sq rows against a chain of chunks (Sk, mask, dist0) with one pstride, slopes of a kind, and the
# lowp_model case fields (head dim, dtype, batch / heads, layout) that seed and shape the inputs.
BF16, FP16 = torch.bfloat16, torch.float16
FAR = 3_000_000


def slopes_for(kind, B, H):
    """fp32 [B, H] slopes of a kind: "std" (flash-attn's), "large" (0.5 .. 1), "tiny" (1e-5), "zero", "neg" (the
    standard ones with the first head's at -0.25) or "bh" (per (batch, head))."""
    std = mo.std_slopes(H).view(1, H).expand(B, H)
    if kind == "std":
        return std.contiguous()
    if kind == "large":
        return torch.linspace(0.5, 1.0, H).view(1, H).expand(B, H).contiguous()
    if kind == "tiny":
        return torch.full((B, H), 1e-5)
    if kind == "zero":
        return torch.zeros(B, H)
    if kind == "neg":
        s = std.clone()
        s[:, 0] = -0.25
        return s
    assert kind == "bh", kind
    return mo.slopes_for(B, H, True, seed=5)


def _mask_id(m):
    if m is None:
        return ""
    if m[0] == "causal_offset":
        return f"c{m[1]}"
    return f"b{m[1]}_{m[2]}"


def acase(sq, chunks, ps=1, slopes="std", D=128, dtype=BF16, B=1, H=2, Hkv=None, layout="flash", tag=""):
    """chunks: [(Sk, mask, dist0)] with mask None, ("causal_offset", off) or ("band", lo, hi)."""
    ch = "+".join(f"{_mask_id(m)}d{d0}" for _, m, d0 in chunks) if len(chunks) <= 3 else f"d{chunks[0][2]}"
    c = lm._case(sq, [(sk, None) for sk, _, _ in chunks], D, dtype, B=B, H=H, Hkv=Hkv, layout=layout,
                 tag=f"alibi_{tag}p{ps}_{slopes}_{ch}_")
    c.update(masks=[m for _, m, _ in chunks], dist0s=[d0 for _, _, d0 in chunks], ps=ps, slopes=slopes)
    return c


def view_chain(sizes, dist0, ps, causal=False):
    """Chunks of one problem: keys of chunk c start sum(sizes[:c]) keys later, so dist0 drops by ps per key; causal:
    the causal mask where d >= 0 (dist0 a multiple of ps)."""
    out, k0 = [], 0
    for sk in sizes:
        d0 = dist0 - ps * k0
        out.append((sk, ("causal_offset", d0 // ps) if causal else None, d0))
        k0 += sk
    return out


def _sweep():
    cs = []
    dts = [(128, BF16), (64, FP16), (64, BF16), (128, FP16)]
    # sign edges: per pstride, a chain whose chunks put tile (0, 0)'s dmin on 0, -1 and -pstride, and one whose chunks
    # put its dmax on 0, 1 and pstride (a chunk is any view: its dist0 is its own)
    shapes = [(129, 257, 128, 383), (65, 513, 255, 1), (255, 127, 63, 129), (383, 64, 513, 257), (63, 129, 257, 65)]
    for i, ps in enumerate((1, 2, 3, 4, 8)):
        sq, a, b, c = shapes[i]
        D, dt = dts[i % 4]
        lo = [127 * ps, 127 * ps - 1, 126 * ps]   # dmin 0, -1, -ps
        hi = [-63 * ps, -63 * ps + 1, -62 * ps]   # dmax 0, 1, ps
        cs.append(acase(sq, [(a, None, lo[0]), (b, None, lo[1]), (c, None, lo[2])], ps, "large", D, dt, tag="dmin_"))
        D, dt = dts[(i + 1) % 4]
        cs.append(acase(sq, [(b, None, hi[0]), (c, None, hi[1]), (a, None, hi[2])], ps, "large" if i < 3 else "std",
                        D, dt, tag="dmax_"))
    # the same edges one tile row / column further on, and at +-64 ps and +-128 ps, +-1 and +-ps, one chunk each
    for i, (ps, d0) in enumerate([(1, 64), (1, -64), (1, 128 + 1), (1, -128 - 1), (2, 2 * 64 + 2), (2, -2 * 128 - 2),
                                  (3, 3 * 128 - 1), (3, -3 * 64 + 3), (4, 4 * 127 + 4 * 64), (8, -8 * 63 - 8 * 64 + 8),
                                  (8, 8 * 127 - 8 * 64 - 1), (4, -4 * 63 + 4 * 128 + 1)]):
        D, dt = dts[i % 4]
        sq, sk = [(257, 513), (383, 255), (129, 383), (513, 129), (255, 257), (65, 513)][i % 6]
        cs.append(acase(sq, [(sk, None, d0)], ps, ["std", "large"][i % 2], D, dt))
    # d never 0: pstride does not divide dist0, across and beside d = 0
    cs.append(acase(257, [(257, None, 5), (129, None, 3 * 127 + 1)], 3, "large", 128, BF16, tag="nozero_"))
    cs.append(acase(129, [(383, None, -8 * 63 - 3)], 8, "std", 64, FP16, tag="nozero_"))
    # one row / one key
    cs.append(acase(1, [(513, None, 200)], 1, "large", 128, FP16))
    cs.append(acase(383, [(1, None, -127)], 2, "std", 64, BF16))
    # causal masks on the edges: views of one causal problem (d >= 0 visible), and offsets that do not meet d = 0
    for i, ps in enumerate((1, 2, 4)):
        D, dt = dts[i % 4]
        cs.append(acase(257, [(383, ("causal_offset", 127), 127 * ps)], ps, "large", D, dt, tag="causal_"))
        cs.append(acase(129, view_chain([128, 129], 128 * ps, ps, causal=True), ps, "std", D, dt, tag="causal_"))
    cs.append(acase(255, [(257, ("causal_offset", 1), 64)], 1, "large", 128, FP16, tag="causal_"))
    cs.append(acase(129, [(513, ("causal_offset", -64), -63)], 1, "std", 64, BF16, tag="causal_"))
    # band lower edge with ALiBi (every driver call runs the band launches)
    cs.append(acase(257, [(257, ("band", -100, 0), 0)], 1, "large", 128, BF16, tag="band_"))
    cs.append(acase(200, [(383, ("band", -64, 63), 127)], 2, "std", 64, FP16, tag="band_"))
    cs.append(acase(129, [(257, ("band", 150, None), 0)], 1, "std", 128, FP16, tag="band_"))  # rows from 107 dead
    # distance: near->far, far->near, far->far and 16-chunk chains, views of one problem, at large slopes
    for D, dt in [(128, BF16), (64, FP16)]:
        cs.append(acase(129, [(257, None, 100), (128, None, FAR)], 1, "large", D, dt, tag="nearfar_"))
        cs.append(acase(129, [(257, None, FAR), (200, None, 60)], 1, "large", D, dt, tag="farnear_"))
        cs.append(acase(255, view_chain([128, 129], FAR, 1), 1, "large", D, dt, tag="farfar_"))
        cs.append(acase(129, view_chain([64] * 16, -FAR + 1024, 2), 2, "large", D, dt, tag="farfar_"))
        cs.append(acase(129, view_chain([64] * 16, 600, 1), 1, "std", D, dt, tag="chain16_"))
    cs.append(acase(129, [(257, None, -40), (255, None, -FAR - 7)], 3, "large", 128, BF16, tag="nearfar_"))
    cs.append(acase(65, view_chain([128, 64, 129], 2 ** 24 + 3, 1), 1, "large", 128, BF16, tag="2p24_"))
    cs.append(acase(129, [(257, None, -(2 ** 24) - 5)], 1, "std", 64, FP16, tag="2p24_"))
    # slopes: tiny, zero, negative, per (batch, head)
    cs.append(acase(129, [(257, None, 100), (128, None, FAR)], 1, "tiny", 128, BF16))
    cs.append(acase(257, [(255, None, 0)], 1, "tiny", 64, FP16))
    cs.append(acase(129, [(257, None, 60), (129, None, -200)], 1, "zero", 128, FP16))
    cs.append(acase(255, [(257, None, 40), (129, None, 1000)], 1, "neg", 128, BF16))
    cs.append(acase(129, [(383, ("causal_offset", 254), 254)], 1, "neg", 64, FP16))
    cs.append(acase(129, [(257, None, 127), (128, None, FAR)], 2, "bh", 128, BF16, B=2))
    cs.append(acase(255, [(129, None, -63)], 1, "bh", 64, FP16, B=2))
    # grouped-query attention, a distinct slope per query head
    for i, hkv in enumerate((4, 2, 1)):
        D, dt = dts[i % 4]
        cs.append(acase(129, [(257, None, 127 - 64 * i)], 1, "large", D, dt, H=8, Hkv=hkv))
    cs.append(acase(255, [(257, ("causal_offset", 0), 0)], 4, "std", 128, FP16, H=4, Hkv=1))
    # layouts
    for D, dt in [(128, FP16), (64, BF16)]:
        cs.append(acase(129, [(257, ("causal_offset", 127), 127)], 1, "std", D, dt, B=2, layout="bstride"))
        cs.append(acase(255, [(129, None, -64), (128, None, FAR)], 2, "large", D, dt, layout="normal"))
        cs.append(acase(129, [(257, None, 0)], 1, "bh", D, dt, B=2, H=4, Hkv=2, layout="bstride"))
    ids = [c["id"] for c in cs]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    return cs


ALIBI_SWEEP = _sweep()


def _pick(tag, dtype, ps=None, H=None):
    """The id of the first sweep case with this tag (after "alibi_"), dtype, pstride and head count."""
    for c in ALIBI_SWEEP:
        if c["id"].startswith("alibi_" + tag) and c["dtype"] == dtype and (ps is None or c["ps"] == ps) and \
                (H is None or c["H"] == H):
            return c["id"]
    raise LookupError((tag, dtype, ps, H))


# per mutant: one bf16 and one fp16 case of the sweep on which the fault is live
MUTANT_CASES = {
    "sign_dmin_fwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "sign_dmax_fwd": [_pick("dmax_", BF16, 2), _pick("dmax_", FP16, 1)],
    "sign_dmin_bwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "sign_dmax_bwd": [_pick("dmax_", BF16, 2), _pick("dmax_", FP16, 1)],
    "key_term_no_pstride": [_pick("dmin_", BF16, 3), _pick("dmin_", FP16, 2)],
    "bwd_gqa_first_head": [_pick("p1_large", BF16, 1, H=8), _pick("p1_large", FP16, 1, H=8)],
    "carried_not_lowered": [_pick("nearfar_", BF16, 1), _pick("nearfar_", FP16, 1)],
    "dist0_plus1_fwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
    "dist0_plus1_bwd": [_pick("dmin_", BF16, 1), _pick("dmin_", FP16, 2)],
}


def make_alibi_inputs(case, device="cpu"):
    """``lowp_model.make_inputs`` of the case plus its masks and ``alibis[c] = (slopes fp32 [B, H], dist0,
    pstride)`` on ``device``."""
    x = lm.make_inputs(case, device)
    x["masks"] = list(case["masks"])
    slopes = slopes_for(case["slopes"], case["B"], case["H"]).to(device)
    x["alibis"] = [(slopes, d0, case["ps"]) for d0 in case["dist0s"]]
    return x


def dref_source(sq, sk, dist0, pstride):
    """[sq] str per row: "key0" (d < 0 throughout), "keylast" (d > 0 throughout) or "zero" (dref = 0)."""
    hi = pstride * torch.arange(sq, dtype=torch.int64) + int(dist0)
    lo = hi - pstride * (sk - 1)
    return ["key0" if h < 0 else "keylast" if l > 0 else "zero" for h, l in zip(hi.tolist(), lo.tolist())]


def tile_classes(case):
    """The sign classes the case's tiles hit (both kernels classify 64 x 128 tiles), as a set of tuples:
    ("dmin", value, ps) for dmin in {0, -1, -ps}, ("dmax", value, ps) for dmax in {0, 1, ps}, ("cross", ps),
    ("nozero", ps) for a crossing tile where ps does not divide dist0, and ("dref", source) per row."""
    out = set()
    ps = case["ps"]
    sk_of = [sk for sk, _ in case["chunks"]]
    for sk, d0 in zip(sk_of, case["dist0s"]):
        for R in range(0, case["sq"], lm.TILE_M):
            for K in range(0, sk, lm.TILE_N):
                dmin = ps * (R - K - (lm.TILE_N - 1)) + d0
                dmax = ps * (R + lm.TILE_M - 1 - K) + d0
                if dmin in (0, -1, -ps):
                    out.add(("dmin", dmin, ps))
                if dmax in (0, 1, ps):
                    out.add(("dmax", dmax, ps))
                if dmin < 0 < dmax:
                    out.add(("cross", ps))
                    if d0 % ps:
                        out.add(("nozero", ps))
        out.update(("dref", s) for s in dref_source(case["sq"], sk, d0, ps))
    return out
