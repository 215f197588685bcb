"""ALiBi in the 16-bit error model (tests/lowp_alibi.py), without a GPU.

* Unmutated: the model, standing in for the ALiBi kernels, passes the comparator against the fp64 ALiBi oracle on
  every case of the ALiBi edge sweep (tests/test_gpu_alibi_edges.py runs the same cases on the kernels).
* Mutants: each realistic fault of ``lowp_alibi.ALIBI_MUTANTS``, injected into the model, is rejected -- on a bf16 and
  on an fp16 case where it is live.  A mutant that passes means the comparator is too loose.
* Coverage: the sweep's tiles (64 rows x 128 keys, as both kernels classify them) hit every sign edge at every
  pstride, crossing tiles with and without d = 0, every source of a row's reference distance, and carried states
  whose reference is lowered and left alone -- so that an edit of the sweep cannot drop an edge unnoticed.
"""
import pytest
import torch

import lowp_alibi as la
import lowp_model as lm

_BY_ID = {c["id"]: c for c in la.ALIBI_SWEEP}
BF16, FP16 = torch.bfloat16, torch.float16
MUTANT_CASES = la.MUTANT_CASES


def run_case(case, mutant=None, device="cpu"):
    x = la.make_alibi_inputs(case, device)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"])
    got = lm.lowp_chain(*args, mutant=mutant, alibis=x["alibis"])
    ref = lm.oracle_chain(*args, alibis=x["alibis"])
    model = got if mutant is None else lm.lowp_chain(*args, alibis=x["alibis"])
    absmax = la.absmax_prefix(x["q"], x["ks"], x["scale"], x["masks"], x["alibis"])
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)


@pytest.mark.parametrize("case", la.ALIBI_SWEEP, ids=[c["id"] for c in la.ALIBI_SWEEP])
def test_unmutated_model_passes(case):
    run_case(case)


def test_every_mutant_has_cases():
    assert set(MUTANT_CASES) == set(la.ALIBI_MUTANTS)
    for ids in MUTANT_CASES.values():
        assert {_BY_ID[i]["dtype"] for i in ids} == {BF16, FP16}


@pytest.mark.parametrize("mutant,case_id", [(m, i) for m in la.ALIBI_MUTANTS for i in MUTANT_CASES[m]],
                         ids=[f"{m}-{'bf16' if 'bf16' in i else 'fp16'}" for m in la.ALIBI_MUTANTS
                              for i in MUTANT_CASES[m]])
def test_mutant_is_rejected(mutant, case_id):
    with pytest.raises(AssertionError):
        run_case(_BY_ID[case_id], mutant)


def test_sweep_covers_every_alibi_edge():
    hit = set()
    for c in la.ALIBI_SWEEP:
        hit |= la.tile_classes(c)
    want = set()
    for ps in (1, 2, 3, 4, 8):
        want |= {("dmin", 0, ps), ("dmin", -1, ps), ("dmin", -ps, ps), ("dmax", 0, ps), ("dmax", 1, ps),
                 ("dmax", ps, ps), ("cross", ps)}
    want |= {("nozero", ps) for ps in (2, 3, 8)}
    want |= {("dref", "key0"), ("dref", "keylast"), ("dref", "zero")}
    assert not want - hit, f"the ALiBi sweep misses {sorted(want - hit, key=str)}"
    # carried states: some live rows get a lowered reference, some with dref > 0 keep theirs
    info = {}
    for c in la.ALIBI_SWEEP:
        if len(c["chunks"]) > 1:
            x = la.make_alibi_inputs(c)
            lm.lowp_chain(x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], alibis=x["alibis"], info=info)
    assert info.get("lowered", 0) > 0 and info.get("kept", 0) > 0, info
    # the far cases: beyond 2^24 (the loader's fp32 row term inexact), and far chains at slopes of 0.5 and more
    assert any(abs(d) > 2 ** 24 for c in la.ALIBI_SWEEP for d in c["dist0s"])
    assert any(c["slopes"] == "large" and min(abs(d) for d in c["dist0s"]) >= la.FAR - 2048 for c in la.ALIBI_SWEEP)
