"""The band edge sweep of the 16-bit model and comparator of ``tests/lowp_model.py``.

The band ``("band", lo, hi)`` (key b visible to row a iff a + lo <= b <= a + hi, None: open side) is what the tile
kernels' band mask computes; ``lowp_model`` models it, with its causal mutants acting on the band's upper edge and the
faults of ``BAND_MUTANTS`` on its lower edge, through the kernels' index arithmetic restated there
(``fwd_trip_count``, ``fwd_first_tile``, ``bwd_q_range``, ``host_lower``).

``BAND_SWEEP`` is the band edge sweep (tests/test_gpu_window.py runs it on the kernels, tests/test_lowp_band.py on
the model); ``band_tile_classes`` names the edges of the kernels' tiles a case reaches, by the kernels' own index
arithmetic, so that an edit of the sweep cannot drop an edge unnoticed.
"""
from __future__ import annotations

import torch

import lowp_model as lm
from lowp_model import TILE_F, TILE_M, TILE_N, bwd_q_range, fwd_first_tile, fwd_trip_count, host_lower

# One realistic fault each at the band's lower edge.  "_fwd" / "_bwd": only that kernel has the fault.
BAND_MUTANTS = (
    "band_lo_plus1_fwd",            # forward lets the key one below the band through
    "band_lo_plus1_bwd",            # backward does the same
    "band_i_end_short",             # backward: every key block skips the last Q block it should visit (i_end one short)
    "band_lo_minus1_fwd",           # forward drops the band's lowest key a + lo
    "band_lo_minus1_bwd",           # backward does the same
    "band_first_tile_ceil_fwd",     # fwd_first_tile rounds up: the partial first tile of every warpgroup is lost
    "band_wg0_from_wg1_fwd",        # the first warpgroup starts at the second warpgroup's first tile
    "band_need_lo_first_row_bwd",   # need_lo decided from the Q block's first row (q0 + lo > k0), not its last
    "band_drop_at_2_minus_sq",      # the host drops a lower edge of 2 - Sq, which still masks key 0 of row Sq - 1
    "band_clamp_sk_minus1",         # the host clamps lo > Sk to Sk - 1 (row 0 then sees key Sk - 1)
)

# --------------------------------------------------------------------------- #
# the band edge sweep
# --------------------------------------------------------------------------- #
# A case: Sq rows against a chain of chunks (Sk, lo, hi), with the lowp_model case fields (head dim, dtype, key bias,
# batch / heads, layout) that seed and shape the inputs.  The case id carries the bands, so the inputs of a case do
# not change when cases are added around it.
BF16, FP16 = torch.bfloat16, torch.float16
DTS = [(128, BF16), (64, FP16), (64, BF16), (128, FP16)]


def bcase(sq, chunks, D=128, dtype=BF16, bias=None, B=1, H=2, Hkv=None, layout="flash", tag=""):
    """chunks: [(Sk, lo, hi)] with lo / hi None for an open side."""
    if len(chunks) > 3:
        sk, lo, hi = chunks[0]
        ch = f"{len(chunks)}x{sk}b{lo}_{hi}"
    else:
        ch = "+".join(f"{sk}b{lo}_{hi}" for sk, lo, hi in chunks)
    c = lm._case(sq, [(sk, None) for sk, _, _ in chunks], D, dtype, bias=bias, B=B, H=H, Hkv=Hkv, layout=layout,
                 tag=f"band_{tag}{ch}_")
    c["masks"] = [("band", lo, hi) for _, lo, hi in chunks]
    return c


def view_chain(sizes, lo, hi):
    """Chunks of one windowed problem: the band (lo, hi) of the first chunk, shifted down by each chunk's start."""
    out, k0 = [], 0
    for sk in sizes:
        out.append((sk, None if lo is None else lo - k0, None if hi is None else hi - k0))
        k0 += sk
    return out


def _sweep():
    cs = []
    # the chunk cases the window tests began with (ids, and so inputs, unchanged)
    cs += [bcase(257, [(257, -5, 0)]),                      # causal window of 6 keys: inside one tile
           bcase(257, [(257, -100, 0)], 64, FP16),          # crosses 128-key tiles and 64-row blocks
           bcase(383, [(383, -30, 30)]),                    # two-sided, narrower than a warpgroup's 64 rows
           bcase(383, [(383, 0, 0)], 64, BF16),             # the diagonal only
           bcase(255, [(513, 129, 200)], 128, FP16),        # above the diagonal, Sq != Sk
           bcase(129, [(257, 200, None)]),                  # lower edge only; rows from 57 on see nothing
           bcase(130, [(1, -3, 2)], 64, FP16),              # one key
           bcase(65, [(300, -64, 63)], 128, BF16),          # ragged
           bcase(200, [(500, 150, 290)], 128, BF16, H=4, Hkv=2),   # GQA
           bcase(200, [(333, -40, 40)], 64, FP16, H=4, Hkv=1),     # MQA
           bcase(257, [(257, -70, 10)], 128, BF16, bias="randn"),  # key bias with a window
           bcase(129, [(257, -64, 128)], 64, FP16, bias="edge_inf"),
           bcase(200, [(128, 0 - 60, 0), (128, -128 - 60, -128), (100, -256 - 60, -256)], 128, BF16, tag="chain_"),
           bcase(129, [(64, 300, None), (128, -64, 0), (200, -190, -100)], 64, FP16, tag="dead1st_")]
    # the forward's lower-edge phase: (r0 + lo) % 128 in {127, 0, 1} for a warpgroup row r0, lo of both signs, band
    # widths 1, 63/64/65, 127/128/129 and open; Sq % 64 in {1, 63}, Sk % 128 in {1, 127}
    phase = [(257, 513, -1, -1),      # width 1; r0 128: 127.  Backward: q_last % 64 == 0, causal and lower on a pair
             (257, 513, 127, 189),    # width 63; r0 0: 127
             (255, 383, -64, -1),     # width 64; r0 64: 0.  Backward: q_last % 64 == 63
             (257, 513, 128, 192),    # width 65; r0 0: 0
             (255, 383, -63, 63),     # width 127; r0 64: 1.  Backward: need_lo boundary 0
             (257, 513, 129, 256),    # width 128; r0 0: 1
             (255, 383, -65, 63),     # width 129; r0 192: 127
             (257, 513, 1, None),     # open; r0 0: 1
             (255, 383, -128, None),  # open; r0 128: 0
             (129, 257, 128, 128),    # width 1 above the diagonal; r0 0: 0
             (255, 383, 2, 100),      # backward: need_lo boundary 1 (q0 64, k0 128)
             (65, 513, 150, 200)]     # key blocks 0 and 3 idle around the working 1 and 2
    for i, (sq, sk, lo, hi) in enumerate(phase):
        D, dt = DTS[i % 4]
        cs.append(bcase(sq, [(sk, lo, hi)], D, dt, tag="phase_"))
    # host-side lower edges: 1 - Sq (dropped), 2 - Sq (masks key 0 of the last row only), Sk, > Sk (clamped)
    cs.append(bcase(129, [(257, -128, 5)], 128, BF16, tag="host_"))
    cs.append(bcase(129, [(257, -127, 5)], 64, FP16, tag="host_"))
    cs.append(bcase(5, [(3, -3, None)], 128, BF16, tag="host_"))
    cs.append(bcase(63, [(65, -61, None)], 64, FP16, tag="host_"))
    cs.append(bcase(129, [(257, 257, None)], 64, BF16, tag="host_"))
    cs.append(bcase(65, [(129, 200, None)], 128, FP16, tag="host_"))
    cs.append(bcase(129, [(257, 300, 400)], 128, BF16, tag="host_"))
    # carried state: the kernel's CTA with no tile (t0 == n_tiles) keeps the state, lower edges Sk and > Sk in a chain
    for D, dt in [(128, FP16), (64, BF16)]:
        cs.append(bcase(257, [(257, -20, 40), (128, 128, None), (129, 400, None)], D, dt, tag="keep_"))
    # a row whose first visited tile lies wholly below its edge, entering with m = -inf and with a carried m
    cs.append(bcase(257, [(129, -300, -100), (257, -1, 30)], 128, BF16, tag="below_"))
    cs.append(bcase(257, [(64, -50, 0), (257, -65, -1)], 64, FP16, tag="below_"))
    # chains of views of one windowed problem: 16 chunks of 64 keys (most outside most rows' windows, rows dead in
    # the first chunks and revived), and rows alive that see nothing in the last chunk
    for D, dt in [(128, BF16), (64, FP16)]:
        cs.append(bcase(129, view_chain([64] * 16, 1024 - 129 - 200, 1024 - 129), D, dt, tag="chain16_"))
        cs.append(bcase(255, view_chain([256, 128], -200, -50), D, dt, tag="blindlast_"))
    cs.append(bcase(129, view_chain([128, 129, 128], 100, None), 128, FP16, tag="revive_"))
    # deterministic mode: Q blocks whose first visiting key block x_min >= 1, with >= 3 visiting key blocks
    cs.append(bcase(129, [(513, 100, None)], 128, BF16, H=4, Hkv=2, tag="det_"))
    cs.append(bcase(193, [(513, 70, 400)], 64, FP16, H=8, Hkv=2, tag="det_"))
    cs.append(bcase(129, [(513, 130, None)], 64, BF16, H=4, Hkv=1, tag="det_"))
    cs.append(bcase(129, [(513, 100, 420)], 128, FP16, H=2, Hkv=1, tag="det_"))
    # key bias: -inf on the band's edge keys, rows whose whole band is masked by the bias
    cs.append(bcase(257, [(257, -1, 0)], 128, FP16, bias="edge_inf", tag="bias_"))
    cs.append(bcase(255, [(383, -40, -10)], 64, BF16, bias="tile_inf", tag="bias_"))
    cs.append(bcase(257, [(383, 1, 126)], 128, BF16, bias="edge_inf", tag="bias_"))
    # layouts with B = 2
    cs.append(bcase(257, [(383, -63, 1)], 128, FP16, B=2, layout="normal", tag="layout_"))
    cs.append(bcase(255, [(257, -1, 64), (129, -200, -128)], 64, BF16, B=2, layout="bstride", tag="layout_"))
    cs.append(bcase(129, [(257, 64, 191)], 64, FP16, B=2, H=4, Hkv=2, tag="layout_"))
    cs.append(bcase(129, [(257, -65, 0)], 128, BF16, B=2, layout="bstride", bias="randn", tag="layout_"))
    ids = [c["id"] for c in cs]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    return cs


BAND_SWEEP = _sweep()
_BY_ID = {c["id"]: c for c in BAND_SWEEP}


def _pick(prefix, dtype):
    """The id of the first sweep case whose id starts with ``band_`` + prefix, of this dtype."""
    for c in BAND_SWEEP:
        if c["id"].startswith("band_" + prefix) and c["dtype"] == dtype:
            return c["id"]
    raise LookupError((prefix, dtype))


# per mutant: one bf16 and one fp16 case of the sweep on which the fault is live
MUTANT_CASES = {
    "band_lo_plus1_fwd": [_pick("383b-30_30", BF16), _pick("257b-100_0", FP16)],
    "band_lo_plus1_bwd": [_pick("383b-30_30", BF16), _pick("257b-100_0", FP16)],
    "band_i_end_short": [_pick("383b-30_30", BF16), _pick("257b-100_0", FP16)],
    "band_lo_minus1_fwd": [_pick("383b-30_30", BF16), _pick("257b-100_0", FP16)],
    "band_lo_minus1_bwd": [_pick("383b-30_30", BF16), _pick("257b-100_0", FP16)],
    "band_first_tile_ceil_fwd": [_pick("phase_513b-1_-1", BF16), _pick("phase_513b127_189", FP16)],
    "band_wg0_from_wg1_fwd": [_pick("phase_513b-1_-1", BF16), _pick("phase_513b127_189", FP16)],
    "band_need_lo_first_row_bwd": [_pick("phase_513b-1_-1", BF16), _pick("phase_513b127_189", FP16)],
    "band_drop_at_2_minus_sq": [_pick("host_3b-3_None", BF16), _pick("host_65b-61_None", FP16)],
    "band_clamp_sk_minus1": [_pick("host_257b300_400", BF16), _pick("host_129b200_None", FP16)],
}


def make_band_inputs(case, device="cpu"):
    """``lowp_model.make_inputs`` of the case with its band masks, on ``device``."""
    x = lm.make_inputs(case, device)
    x["masks"] = list(case["masks"])
    return x


def _neg_inf_keys(case, sk, c):
    """[B, H, Sk] bool: the keys of chunk c the case's key bias sets to -inf (lowp_model.make_inputs)."""
    kind, B, H = case["bias"], case["B"], case["H"]
    m = torch.zeros(B, H, sk, dtype=torch.bool)
    if kind == "tile_inf":
        m[..., 128:256] = True
    elif kind == "edge_inf":
        m[..., [j for j in (127, 128, sk - 1) if j < sk]] = True
    elif kind == "dead_rows":
        m[..., :64] = True
    elif kind == "head_dead":
        m[:, -1] = True
    return m


def band_tile_classes(case):
    """The edge classes the case reaches, as a set of tuples, from the kernels' index arithmetic per chunk:

    forward (128-row CTAs of two 64-row warpgroups, 128-key tiles): ("fwd_lo_phase", (r0 + lo) % 128 in {127, 0, 1},
    sign of lo) for a warpgroup row r0 with 0 <= r0 + lo < Sk; ("width", hi - lo + 1 or "open"); ("wg1_later_tile",)
    when a CTA's second warpgroup starts in a later tile than its first; ("wg0_ends_earlier",) when a causal CTA's
    first warpgroup ends in an earlier tile; ("cta_no_tile", "fresh" / "carried") for a CTA with t0 == n_tiles;
    ("below_edge", "fresh" / "carried") for a row whose first visited tile lies wholly below its edge;
    backward (128-key blocks, 64-row Q blocks): ("q_last", q_last % 64 in {0, 63}) for a key block whose last
    visiting Q block is cut by the band; ("need_lo", q0 + 63 + lo - k0 in {0, 1}) on a visited pair;
    ("causal_and_lo",) on a pair both masks apply to; ("idle_around_work",) for a launch with key blocks that have
    no Q block both below and above the working ones (both bounds grow with k0, so idle blocks sit only there);
    ("det_x_min", G, "mqa" / "gqa") for a Q block with x_min >= 1 and >= 3 visiting key blocks;
    host: ("host_lo", "1-Sq" / "2-Sq" / "Sk" / ">Sk" / "=causal");
    chains: ("chain16",), ("revived",) (dead after the first chunk, alive at the end), ("blind_last",) (alive before
    the last chunk, sees nothing in it); key bias: ("bias_edge",) -inf on a row's lowest or highest band key,
    ("bias_whole_band",) a row whose every band key is -inf;
    shapes: ("sq_mod64", 1 / 63), ("sk_mod128", 1 / 127), ("dtype", name, D), ("layout", layout, B)."""
    out = set()
    sq, B, H, Hkv = case["sq"], case["B"], case["H"], case["Hkv"]
    G = H // Hkv
    out.add(("dtype", "bf16" if case["dtype"] == BF16 else "fp16", case["D"]))
    out.add(("layout", case["layout"], B))
    if sq % 64 in (1, 63):
        out.add(("sq_mod64", sq % 64))
    alive = torch.zeros(sq, dtype=torch.bool)  # rows that saw a key in an earlier chunk (visibility only)
    n = len(case["chunks"])
    if n == 16 and all(sk == 64 for sk, _ in case["chunks"]):
        out.add(("chain16",))
    alive_after = []
    for c, ((sk, _), (_, lo0, hi)) in enumerate(zip(case["chunks"], case["masks"])):
        if sk % 128 in (1, 127):
            out.add(("sk_mod128", sk % 128))
        if lo0 is not None:
            if lo0 == 1 - sq:
                out.add(("host_lo", "1-Sq"))
            elif lo0 == 2 - sq:
                out.add(("host_lo", "2-Sq"))
            elif lo0 == sk:
                out.add(("host_lo", "Sk"))
            elif lo0 > sk:
                out.add(("host_lo", ">Sk"))
            if hi is not None and lo0 == hi:
                out.add(("host_lo", "=causal"))
        out.add(("width", "open" if hi is None or lo0 is None else hi - lo0 + 1))
        vis = lm.visible(sq, sk, ("band", lo0, hi))
        sees = vis.any(1)
        lo = host_lower(sq, sk, lo0)
        carried = "carried" if c > 0 else "fresh"
        if lo is not None:
            sign = "pos" if lo > 0 else "neg" if lo < 0 else "zero"
            # forward
            for row0 in range(0, sq, TILE_F):
                n_all = max(fwd_trip_count(row0, sq, sk, hi), fwd_trip_count(row0 + 64, sq, sk, hi))
                t0 = min(fwd_first_tile(row0, lo), n_all)
                if t0 == n_all:
                    out.add(("cta_no_tile", carried))
                if row0 + 64 < sq and fwd_first_tile(row0 + 64, lo) > fwd_first_tile(row0, lo) and \
                        fwd_first_tile(row0 + 64, lo) < fwd_trip_count(row0 + 64, sq, sk, hi):
                    out.add(("wg1_later_tile",))
                if hi is not None and row0 + 64 < sq and \
                        0 < fwd_trip_count(row0, sq, sk, hi) < fwd_trip_count(row0 + 64, sq, sk, hi):
                    out.add(("wg0_ends_earlier",))
                for r0 in (row0, row0 + 64):
                    if r0 >= sq:
                        continue
                    if 0 <= r0 + lo < sk and (r0 + lo) % 128 in (127, 0, 1):
                        out.add(("fwd_lo_phase", (r0 + lo) % 128, sign))
                    my0 = fwd_first_tile(r0, lo)
                    if my0 < fwd_trip_count(r0, sq, sk, hi):
                        for a in range(r0, min(r0 + 64, sq)):
                            if a + lo >= (my0 + 1) * TILE_N and bool(sees[a]):
                                out.add(("below_edge", "carried" if c > 0 and bool(alive[a]) else "fresh"))
            # backward
            nq = (sq + TILE_M - 1) // TILE_M
            work = []
            for k0 in range(0, sk, TILE_N):
                ib, ie = bwd_q_range(k0, sq, sk, lo, hi)
                work.append(ie > ib)
                q_last = min(k0 + TILE_N - 1, sk - 1) - lo
                if ie > ib and 0 <= q_last < sq and q_last % 64 in (0, 63):
                    out.add(("q_last", q_last % 64))
                for i in range(ib, ie):
                    q0 = i * TILE_M
                    need_lo = q0 + TILE_M - 1 + lo > k0
                    if q0 + TILE_M - 1 + lo - k0 in (0, 1):
                        out.add(("need_lo", q0 + TILE_M - 1 + lo - k0))
                    if need_lo and hi is not None and q0 + hi < k0 + TILE_N - 1:
                        out.add(("causal_and_lo",))
            first = work.index(True) if any(work) else None
            if first is not None and first > 0 and not work[-1]:
                out.add(("idle_around_work",))
            for i in range(nq):
                xs = [x for x in range(len(work)) if bwd_q_range(x * TILE_N, sq, sk, lo, hi)[0] <= i <
                      bwd_q_range(x * TILE_N, sq, sk, lo, hi)[1]]
                x_min = max(0, i * TILE_M + lo) // TILE_N
                if xs and xs[0] == x_min >= 1 and len(xs) >= 3 and G > 1:
                    out.add(("det_x_min", G, "mqa" if Hkv == 1 else "gqa"))
        # key bias on the band's edge keys
        if case["bias"] is not None:
            inf = _neg_inf_keys(case, sk, c)  # [B,H,Sk]
            a = torch.arange(sq)
            for edge in (lo0, hi):
                if edge is None:
                    continue
                j = a + edge
                ok = (j >= 0) & (j < sk)
                if ok.any() and inf[..., j[ok]].any():
                    out.add(("bias_edge",))
            if ((inf.unsqueeze(2) | ~vis).all(-1) & sees).any():  # [B,H,Sq]
                out.add(("bias_whole_band",))
        if c == n - 1 and c > 0 and (alive & ~sees).any():
            out.add(("blind_last",))
        alive = alive | sees
        alive_after.append(alive.clone())
    if n > 1 and (~alive_after[0] & alive_after[-1]).any():
        out.add(("revived",))
    return out

