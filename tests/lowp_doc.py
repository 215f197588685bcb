"""The document edge sweep of the 16-bit model and comparator of ``tests/lowp_model.py``.

A document mask ``("doc", lo, hi, cu, q_pos0, k_pos0, pstride)`` is what the doc tile kernels compute for one launch:
the band ``("band", lo, hi)`` (key b visible to row a iff a + lo <= b <= a + hi, None: open side), and row a (at
position q_pos0 + pstride a) sees key b (at k_pos0 + pstride b) only inside one document ``[cu[d], cu[d + 1])``.
``lowp_model`` models it; the faults of ``DOC_MUTANTS`` act there through the kernels' own index arithmetic, restated
in ``doc_index`` (a fault there is a fault of the model's visibility).

``DOC_SWEEP`` is the document edge sweep (tests/test_gpu_varlen.py runs it on the kernels, tests/test_lowp_doc.py on
the model); ``doc_tile_classes`` names the edges of the kernels' tiles a case reaches, by the kernels' index
arithmetic, so that an edit of the sweep cannot drop an edge unnoticed.
"""
from __future__ import annotations

import torch

import doc_index as di
import lowp_model as lm

# One realistic fault each.  "_fwd" / "_bwd": only that kernel has the fault.
DOC_MUTANTS = (
    "doc_edge_plus1_fwd",           # forward lets the first key of the next document through
    "doc_edge_plus1_bwd",           # backward does the same
    "doc_edge_minus1_fwd",          # forward drops the last key of the row's document
    "doc_edge_minus1_bwd",          # backward does the same
    "doc_range_first_row_fwd",      # a warpgroup's tile range ends at its first row's document
    "doc_i_end_first_key_bwd",      # a key block's i_end from the document of its first key, not its last
    "doc_search_lower_bound",       # the document search finds the first d with cu[d] >= x (both kernels)
    "doc_planner_drop_last_key",    # the planner drops a launch whose rows share a document only with its last key
)

BF16, FP16 = torch.bfloat16, torch.float16


# --------------------------------------------------------------------------- #
# the document edge sweep
# --------------------------------------------------------------------------- #
def dcase(name, sq, chunks, D=128, dtype=BF16, H=2, Hkv=None, cu=None, q_pos0=0, ps=1):
    """chunks: [(Sk, k_pos0, lo, hi)] of rows sq at position q_pos0 + ps a, against documents cu."""
    c = lm._case(sq, [(sk, None) for sk, _, _, _ in chunks], D, dtype, H=H, Hkv=Hkv, tag=f"doc_{name}_")
    c["masks"] = [("doc", lo, hi, tuple(cu), q_pos0, kp, ps) for _, kp, lo, hi in chunks]
    return c


def _sweep():
    cs = []
    # boundaries at tile phases 127/0/1 of 128-row CTAs, 64-row blocks and 128-key tiles; the two warpgroups of CTAs in
    # different documents; GQA for the deterministic turn counters (Q blocks whose x_min >= 1 comes from a document)
    edges = (0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 385)
    cs.append(dcase("phase", 385, [(385, 0, None, 0)], 128, BF16, H=4, Hkv=2, cu=edges))
    cs.append(dcase("phase", 385, [(385, 0, None, None)], 64, FP16, H=4, Hkv=1, cu=edges))
    # several documents (and zero-length ones) inside one tile, with a window
    small = (0, 5, 9, 9, 30, 31, 40, 41, 300, 300, 385)
    cs.append(dcase("small", 385, [(385, 0, -70, 0)], 128, FP16, cu=small))
    cs.append(dcase("small", 385, [(385, 0, -40, 40)], 64, BF16, cu=small))
    # one document over many tiles
    cs.append(dcase("long", 600, [(600, 0, None, None)], 64, BF16, H=4, Hkv=2, cu=(0, 3, 590, 600)))
    cs.append(dcase("long", 600, [(600, 0, None, 0)], 128, FP16, cu=(0, 3, 590, 600)))
    # striped rounds: pstride 2, 4, 8, rows of rank iq against keys of rank jk (causal: c <= a + (iq - jk) // W)
    for W, iq, jk, D, dt in ((2, 1, 0, 128, BF16), (4, 0, 3, 64, FP16), (8, 5, 2, 128, FP16), (8, 2, 5, 64, BF16)):
        T = 300 * W
        cu = (0, 127 * W, 128 * W + 1, 130 * W, 260 * W - 1, T)
        cs.append(dcase(f"striped{W}_{iq}{jk}", 300, [(300, jk, None, (iq - jk) // W)], D, dt, H=4, Hkv=2, cu=cu,
                        q_pos0=iq, ps=W))
    # ring chains (contiguous shards of 256): the rows of shard 1 against the keys of shards 0, 1, 2 -- rows dead in
    # the first chunk and revived in the second; a round that shares its rows' document only at its last key
    for D, dt in ((128, BF16), (64, FP16)):
        cs.append(dcase("revive", 256, [(256, 0, None, None), (256, 256, None, None), (256, 512, None, None)], D, dt,
                        cu=(0, 200, 300, 600, 768), q_pos0=256))
        cs.append(dcase("lastkey", 256, [(256, 0, None, None), (256, 256, None, 0)], D, dt, H=4, Hkv=2,
                        cu=(0, 255, 520, 768), q_pos0=256))
    ids = [c["id"] for c in cs]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    return cs


DOC_SWEEP = _sweep()
_BY_ID = {c["id"]: c for c in DOC_SWEEP}


def make_doc_inputs(case, device="cpu"):
    """``lowp_model.make_inputs`` of the case with its document masks, on ``device``."""
    x = lm.make_inputs(case, device)
    x["masks"] = list(case["masks"])
    return x


def live(case, mutant):
    """Whether the mutant changes what some chunk of the case sees, in either kernel."""
    sq = case["sq"]
    for (sk, _), m in zip(case["chunks"], case["masks"]):
        ref = lm.visible(sq, sk, m)
        if any(not torch.equal(lm._vis_for(sq, sk, m, None, mutant, side), ref) for side in ("fwd", "bwd")):
            return True
    return False


def mutant_cases():
    """Per mutant: the first bf16 and the first fp16 case of the sweep on which it is live."""
    out = {}
    for m in DOC_MUTANTS:
        out[m] = [next((c["id"] for c in DOC_SWEEP if c["dtype"] == dt and live(c, m)), None) for dt in (BF16, FP16)]
    return out


def doc_tile_classes(case):
    """The edge classes the case reaches, as a set of tuples, from the kernels' index arithmetic per chunk:

    ("row_edge", 128 / 64, p) and ("key_edge", p): a document starting at row (key) index i of the launch with
    i % 128 in {127, 0, 1} (i % 64 in {63, 0, 1}); ("docs_in_tile",): three or more documents with keys in one 128-key tile;
    ("doc_spans_tiles",): a document whose keys span three or more tiles; ("zero_length",); ("pstride", W);
    ("wg_split",): a CTA whose two warpgroups' rows lie in different documents; ("dead_row",): a row with no key in
    a launch; ("revived",): a row with no key in the first chunk that sees keys later; ("planner_last_key",): a launch
    whose rows share a document only with its last key; ("flag", "on" / "off"): a backward (key block, Q block) pair
    that crosses a document edge or not; ("det_x_min_doc", "gqa" / "mqa"): a Q block whose first visiting key block
    x_min >= 1 is set by its document; ("dtype", name, D)."""
    out = set()
    sq, H, Hkv = case["sq"], case["H"], case["Hkv"]
    out.add(("dtype", "bf16" if case["dtype"] == BF16 else "fp16", case["D"]))
    alive0 = None
    for c, ((sk, _), m) in enumerate(zip(case["chunks"], case["masks"])):
        _, lo, hi, cu, q_pos0, k_pos0, ps = m
        L = lm.doc_launch(sq, sk, m)
        if ps > 1:
            out.add(("pstride", ps))
        if any(a == b for a, b in zip(cu, cu[1:])):
            out.add(("zero_length",))
        for b in cu[1:-1]:
            r = di.view_index(b, q_pos0, ps, sq)  # the first row of the document that starts at b
            if 0 < r < sq:
                for t in (128, 64):
                    if r % t in (t - 1, 0, 1):
                        out.add(("row_edge", t, r % t))
            k = di.view_index(b, k_pos0, ps, sk)
            if 0 < k < sk and k % 128 in (127, 0, 1):
                out.add(("key_edge", k % 128))
        docs = di.doc_of
        for t0 in range(0, sk, 128):
            ds = {docs(cu, k_pos0 + ps * j) for j in range(t0, min(t0 + 128, sk))}
            if len(ds) >= 3:
                out.add(("docs_in_tile",))
        for d in range(len(cu) - 1):
            lo_k, hi_k = di.view_index(cu[d], k_pos0, ps, sk), di.view_index(cu[d + 1], k_pos0, ps, sk)
            if hi_k > lo_k and (hi_k - 1) // 128 - lo_k // 128 >= 2:
                out.add(("doc_spans_tiles",))
        for row0 in range(0, sq, 128):
            if row0 + 64 < sq:
                last0 = docs(cu, q_pos0 + ps * min(row0 + 63, sq - 1))
                if docs(cu, q_pos0 + ps * (row0 + 64)) > last0:
                    out.add(("wg_split",))
        vis = lm.visible(sq, sk, m)
        sees = vis.any(1)
        if (~sees).any():
            out.add(("dead_row",))
        if c == 0:
            alive0 = sees
        elif (~alive0 & sees).any():
            out.add(("revived",))
        if lm.planner_drops_last_key(sq, sk, m) and vis.any():
            out.add(("planner_last_key",))
        nQ = (sq + 63) // 64
        visits = [[] for _ in range(nQ)]
        for x in range((sk + 127) // 128):
            ib, ie = L.q_blocks(x)
            for i in range(ib, ie):
                visits[i].append(x)
                cross = any(L.staged(a, x) != (0, min(128, sk - x * 128)) for a in range(i * 64, min(i * 64 + 64, sq)))
                out.add(("flag", "on" if cross else "off"))
        if H // Hkv > 1:
            for i in range(nQ):
                band_x = max(0, i * 64 + L.lo) // 128
                if visits[i] and visits[i][0] == L.x_min(i) >= 1 and L.x_min(i) > band_x and len(visits[i]) >= 2:
                    out.add(("det_x_min_doc", "mqa" if Hkv == 1 else "gqa"))
    return out
