"""Packed-document masks in the 16-bit error model (tests/lowp_doc.py), without a GPU.

* Unmutated: the model, standing in for the doc kernels, passes the comparator against the fp64 document oracle on
  every case of the document edge sweep (tests/test_gpu_varlen.py runs the same cases on the kernels).
* Mutants: each realistic fault of ``lowp_doc.DOC_MUTANTS``, injected into the model through the kernels' restated
  index arithmetic, is rejected -- on a bf16 and on an fp16 case where it is live.  A mutant that passes means the
  comparator is too loose.
* Coverage: the sweep reaches every edge of ``lowp_doc.doc_tile_classes`` listed below, so that an edit of the sweep
  cannot drop one unnoticed.
"""
import pytest
import torch

import lowp_doc as ld
import lowp_model as lm

BF16, FP16 = torch.bfloat16, torch.float16
MUTANT_CASES = ld.mutant_cases()


def run_case(case, mutant=None):
    x = ld.make_doc_inputs(case)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got = lm.lowp_chain(*args, mutant=mutant)
    ref = lm.oracle_chain(*args)
    model = got if mutant is None else lm.lowp_chain(*args)
    absmax = [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1]) for c in range(len(x["ks"]))]
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)


@pytest.mark.parametrize("case", ld.DOC_SWEEP, ids=[c["id"] for c in ld.DOC_SWEEP])
def test_unmutated_model_passes(case):
    run_case(case)


def test_every_mutant_has_cases():
    assert set(MUTANT_CASES) == set(ld.DOC_MUTANTS)
    for m, ids in MUTANT_CASES.items():
        assert None not in ids, f"{m} is live on no bf16 or no fp16 case of the sweep"


@pytest.mark.parametrize("mutant,dt", [(m, i) for m in ld.DOC_MUTANTS for i in (0, 1)],
                         ids=[f"{m}-{d}" for m in ld.DOC_MUTANTS for d in ("bf16", "fp16")])
def test_mutant_is_rejected(mutant, dt):
    with pytest.raises(AssertionError):
        run_case(ld._BY_ID[MUTANT_CASES[mutant][dt]], mutant)


# every class of lowp_doc.doc_tile_classes the sweep must reach
WANT = (
    {("row_edge", 128, p) for p in (127, 0, 1)} | {("row_edge", 64, p) for p in (63, 0, 1)}
    | {("key_edge", p) for p in (127, 0, 1)}
    | {("docs_in_tile",), ("doc_spans_tiles",), ("zero_length",), ("wg_split",), ("dead_row",), ("revived",),
       ("planner_last_key",), ("flag", "on"), ("flag", "off")}
    | {("pstride", W) for W in (2, 4, 8)}
    | {("det_x_min_doc", kind) for kind in ("gqa", "mqa")}
    | {("dtype", n, D) for n in ("bf16", "fp16") for D in (64, 128)}
)


def test_sweep_covers_every_document_edge():
    hit = set()
    for c in ld.DOC_SWEEP:
        hit |= ld.doc_tile_classes(c)
    assert not WANT - hit, f"the document sweep misses {sorted(WANT - hit, key=str)}"
