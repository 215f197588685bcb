"""``scale_model.run``, the row-blocked oracle and 16-bit model, on the CPU.

* Agreement: on single-chunk cases of ``SWEEP``, ``BAND_SWEEP``, ``ALIBI_SWEEP`` and ``DOC_SWEEP`` the blocked truth is
  ``oracle_chain`` to fp64 round-off (every field the comparator reads), and the blocked model is ``lowp_chain`` to
  fp32 round-off (O to one 16-bit ulp), far inside the comparator's own row scale for every output.  Row blocks of
  37 and 100 rows divide no case and are shorter than a tile, and cut windows and documents anywhere; a seam makes
  every block a chain of two chunks.
* Teeth: on a problem of 4096 rows and keys with a seam at key 2048 (the kernels' L2 split at S = 65536, scaled
  down 16 times), the comparator rejects a model run with one fault: one key dropped at the seam, one key dropped
  at a window's lower edge, a document edge one key off (or a boundary moved by one position), one 128-key tile
  missing from dQ, one 64-row Q block missing from dV, the state carried across the seam loaded with l = 4.  The
  clean model passes.
"""
import functools

import pytest
import torch

import lowp_alibi as la
import lowp_band as lb
import lowp_doc as ld
import lowp_model as lm
import mask_oracle as mo
import scale_model as sm


def _single(cases, n):
    """Up to n single-chunk cases without a key bias, spread over the sweep, and every such GQA or B = 2 case."""
    one = [c for c in cases if len(c["chunks"]) == 1 and not c.get("bias")]
    pick = one[::max(1, len(one) // n)][:n]
    extra = [c for c in one if (c["Hkv"] != c["H"] or c["B"] > 1) and c not in pick][:2]
    return pick + extra


def _whole(case):
    """The case as one whole call: (inputs, mask, alibi)."""
    if case in la.ALIBI_SWEEP:
        x = la.make_alibi_inputs(case)
        return x, x["masks"][0], x["alibis"][0]
    if case in lb.BAND_SWEEP:
        x = lb.make_band_inputs(case)
    elif case in ld.DOC_SWEEP:
        x = ld.make_doc_inputs(case)
    else:
        x = lm.make_inputs(case)
    return x, x["masks"][0], None


CASES = _single(lm.SWEEP, 4) + _single(lb.BAND_SWEEP, 4) + _single(la.ALIBI_SWEEP, 4) + _single(ld.DOC_SWEEP, 5)
assert any(c["Hkv"] != c["H"] for c in CASES) and any(c["B"] > 1 for c in CASES)


def _close(name, got, want, rtol, atol=0.0):
    got, want = got.detach().double(), want.detach().double()
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin) and torch.equal(got[~fin], want[~fin]), name
    err = (got[fin] - want[fin]).abs()
    lim = rtol * want[fin].abs() + atol * float(want[fin].abs().max() if fin.any() else 0.0)
    assert bool((err <= lim).all()), f"{name}: off by {float((err - lim).max()):.3e} beyond rtol {rtol}"


@pytest.mark.parametrize("block,seam", [(37, False), (100, True)], ids=["b37", "b100-seam"])
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_blocked_agrees_with_whole_chains(case, block, seam):
    x, mask, alibi = _whole(case)
    q, k, v, do, scale = x["q"], x["ks"][0], x["vs"][0], x["do"], x["scale"]
    sk = k.shape[1]
    seams = (sk // 2 + 3,) if seam and sk > 8 else ()
    got = sm.run(q, k, v, do, scale, mask, alibi, block=block, seams=seams)
    assert got["heads"] == list(range(case["H"]))
    t, m = got["truth"], got["model"]
    # the whole rows as one chain, cut at the seam as every block is (the model rounds P per chunk)
    cuts = [0, *seams, sk]
    ks, vs = [k[:, a:b] for a, b in zip(cuts, cuts[1:])], [v[:, a:b] for a, b in zip(cuts, cuts[1:])]
    chunks = [sm.restate(mask, alibi, 0, a) for a in cuts[:-1]]
    masks, alibis = [c[0] for c in chunks], None if alibi is None else [c[1] for c in chunks]
    ref = lm.oracle_chain(q, ks, vs, do, scale, masks, alibis=alibis)
    model = lm.lowp_chain(q, ks, vs, do, scale, masks, alibis=alibis)
    cat = lambda d, n: torch.cat(d[n], 1)  # noqa: E731
    # the truth: fp64 round-off, in every field the comparator reads
    for n in ("o", "lse", "dq"):
        _close(f"truth {n}", t[n], ref[n], 1e-12, 1e-13)
    for n in ("dk", "dv"):
        _close(f"truth {n}", t[n][0], cat(ref, n), 1e-12, 1e-13)
    for n in ("o", "dq", "dk", "dv"):
        _close(f"rss {n}", t["rss"][n], ref["rss"][n], 1e-12, 1e-13)
    for n in ("dq", "dk"):
        _close(f"e32 {n}", t["e32"][n], ref["e32"][n], 1e-12, 1e-13)
    assert t["mag"] == pytest.approx(ref["mag"], rel=1e-15)
    if alibi is None:
        _close("absmax", t["absmax"], lm.scores_absmax(q, ks, scale, masks), 1e-15)
    # the model: lse to fp32 round-off, O in 16 bit nearly everywhere the same
    u = lm.unit_roundoff(q.dtype)
    _close("model lse", m["lse"], model["lse"], 1e-6, 1e-6)
    assert float((m["o"] != model["o"]).double().mean()) < 0.02, "the model's O differs beyond rounding flips"
    # every output far inside the comparator's row bound B |model - ref| + C u rss + FLOOR mag + e32: the two models
    # differ only where a 16-bit rounding of P or dS flips under a different fp32 summation order
    for n, a, b, r in (("o", m["o"], model["o"], ref["o"]), ("dq", m["dq"], model["dq"], ref["dq"]),
                       ("dk", m["dk"][0], cat(model, "dk"), cat(ref, "dk")),
                       ("dv", m["dv"][0], cat(model, "dv"), cat(ref, "dv"))):
        diff = (a.double() - b.double()).norm(dim=-1)
        mag = ref["mag"][n] if n != "o" else float(r.norm(dim=-1).max())
        extra = ref["e32"][n] if n in ("dq", "dk") else 0.0
        bound = lm.B * (b.double() - r).norm(dim=-1) + lm.C * u * ref["rss"][n] + lm.FLOOR * mag + extra
        assert bool((diff <= 0.25 * bound).all()), f"model {n}: {float((diff / bound).max()):.3f} of the row bound"


# --------------------------------------------------------------------------- #
# teeth: faults of the model at a CPU-sized analogue of S = 65536 with its L2 seam
# --------------------------------------------------------------------------- #
S, SEAM, BLOCK, H, HKV, D = 4096, 2048, 512, 2, 1, 64
DT = torch.bfloat16
DOCS = (0, 700, 1500, 2047, 2049, 2900, 4096)  # documents across the seam and across row blocks
WORKLOADS = {
    "window": ("band", -511, 0),                        # flash_attn_func(causal, window_size=(511, 0))
    "causal": ("causal_offset", 0),
    "doc": ("doc", None, 0, DOCS, 0, 0, 1),             # causal inside each document
    "doc_full": ("doc", None, None, DOCS, 0, 0, 1),     # not causal: the next document's first key is a live fault
}


@functools.lru_cache(maxsize=None)
def _inputs():
    g = torch.Generator().manual_seed(4096)
    rn = lambda h: torch.randn(1, S, h, D, generator=g).to(DT)  # noqa: E731
    return rn(H), rn(HKV), rn(HKV), rn(H)


@functools.lru_cache(maxsize=None)
def _clean(work):
    q, k, v, do = _inputs()
    return sm.run(q, k, v, do, D ** -0.5, WORKLOADS[work], block=BLOCK, seams=(SEAM,))


def _as_api(model):
    """A model run as the API would return it: 16-bit O and gradients."""
    return {n: (model[n] if n == "o" else model[n] if n == "dq" else model[n][0]).to(DT) for n in ("o", "dq", "dk", "dv")}


def _check(work, model):
    r = _clean(work)
    lm.assert_api_within_model(f"scale_{work}", _as_api(model), r["truth"], r["model"], DT)


@pytest.mark.parametrize("work", list(WORKLOADS))
def test_clean_model_passes(work):
    _check(work, _clean(work)["model"])


def _faulty(work, mask=None, **kw):
    q, k, v, do = _inputs()
    return sm.run(q, k, v, do, D ** -0.5, mask or WORKLOADS[work], block=BLOCK, seams=(SEAM,), truth=False, **kw)["model"]


AT_SEAM = range(SEAM, SEAM + 1)  # the row block that starts at the seam
FAULTS = [
    # one key no row sees: the first key after the seam (no mutant states a fault at one absolute key)
    ("seam_key_window", "window", dict(drop_keys=(SEAM,))),
    ("seam_key_causal", "causal", dict(drop_keys=(SEAM,))),
    ("seam_key_doc", "doc", dict(drop_keys=(SEAM,))),
    # the window's lowest key a - 511 of every row of one block, in one kernel
    ("band_lo_minus1_fwd", "window", dict(mutant="band_lo_minus1_fwd", mutant_rows=AT_SEAM)),
    ("band_lo_minus1_bwd", "window", dict(mutant="band_lo_minus1_bwd", mutant_rows=AT_SEAM)),
    # a document edge one key off in the kernels' index arithmetic, for the rows of one block
    ("doc_edge_plus1_fwd", "doc_full", dict(mutant="doc_edge_plus1_fwd", mutant_rows=AT_SEAM)),
    ("doc_edge_minus1_fwd", "doc", dict(mutant="doc_edge_minus1_fwd", mutant_rows=AT_SEAM)),
    ("doc_edge_plus1_bwd", "doc_full", dict(mutant="doc_edge_plus1_bwd", mutant_rows=AT_SEAM)),
    ("doc_edge_minus1_bwd", "doc", dict(mutant="doc_edge_minus1_bwd", mutant_rows=AT_SEAM)),
    # dQ of one row block misses the partial of one 128-key tile
    ("dq_missing_key_block", "causal", dict(mutant="dq_missing_key_block", mutant_rows=AT_SEAM)),
    # dV misses one 64-row Q block of one row block
    ("dv_missing_q_block", "causal", dict(mutant="dv_missing_q_block", mutant_rows=AT_SEAM)),
    # the state carried across the seam enters with l = 4
    ("carried_l4_causal", "causal", dict(mutant="carried_l4")),
    ("carried_l4_window", "window", dict(mutant="carried_l4")),
]


@pytest.mark.parametrize("work,kw", [f[1:] for f in FAULTS], ids=[f[0] for f in FAULTS])
def test_fault_at_scale_rejected(work, kw):
    with pytest.raises(AssertionError, match="outside the model bound|max\\|got-ref\\|"):
        _check(work, _faulty(work, **kw))


@pytest.mark.parametrize("moved", [+1, -1])
def test_document_boundary_moved_rejected(moved):
    """The boundary at 2049 (one key past the seam) moved by one position: the model run on those documents."""
    cu = tuple(c + moved if c == 2049 else c for c in DOCS)
    with pytest.raises(AssertionError, match="outside the model bound|max\\|got-ref\\|"):
        _check("doc", _faulty("doc", ("doc", None, 0, cu, 0, 0, 1)))


def test_refuses_split_kv_group():
    q, k, v, do = _inputs()
    with pytest.raises(AssertionError, match="split K/V head"):
        sm.run(q[:, :64], k[:, :64], v[:, :64], do[:, :64], D ** -0.5, heads=[0])


def test_full_fp32_restores_settings():
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("high")
    try:
        with sm.full_fp32():
            assert torch.get_float32_matmul_precision() == "highest"
            assert not torch.backends.cuda.matmul.allow_tf32
        assert torch.get_float32_matmul_precision() == "high"
    finally:
        torch.set_float32_matmul_precision(prev)


def test_key_range_is_what_the_mask_lets_through():
    """``key_range`` of a row block is exactly the keys its rows see, for every mask kind (pstride 2 documents)."""
    masks = [None, ("causal_offset", -70), ("band", -100, 30), ("band", 40, None),
             ("doc", None, 0, (0, 5, 9, 9, 130, 300, 700), 3, 1, 2), ("doc", -50, 50, (0, 200, 210, 600), 0, 0, 1)]
    for mask in masks:
        vis = mo.mask_of(300, 301, mask)
        for r0, r1 in [(0, 37), (37, 74), (100, 228), (290, 300)]:
            k0, k1 = sm.key_range(mask, r0, r1, 301)
            seen = torch.ones(301, dtype=torch.bool) if vis is None else vis[r0:r1].any(0)
            idx = seen.nonzero().flatten().tolist()
            if not idx:
                assert k1 <= k0, (mask, r0, r1)
            else:
                assert k0 <= idx[0] and idx[-1] < k1, (mask, r0, r1, k0, k1, idx[0], idx[-1])
                assert k0 == idx[0] or mask[0] == "doc", (mask, r0, r1)
