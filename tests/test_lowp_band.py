"""The band (sliding-window) mask in the 16-bit error model (tests/lowp_band.py), without a GPU.

* Unmutated: the model, standing in for the band kernels, passes the comparator against the fp64 band oracle on
  every case of the band edge sweep (tests/test_gpu_window.py runs the same cases on the kernels).
* Mutants: each realistic fault of ``lowp_band.BAND_MUTANTS``, injected into the model, is rejected -- on a bf16 and
  on an fp16 case where it is live.  A mutant that passes means the comparator is too loose.
* Coverage: the sweep reaches every edge of the band kernels' tiles, of the host's lower-edge clamps, of the
  deterministic mode's turn counters and of carried states -- so that an edit of the sweep cannot drop an edge
  unnoticed.
"""
import pytest
import torch

import lowp_band as lb
import lowp_model as lm

_BY_ID = {c["id"]: c for c in lb.BAND_SWEEP}
BF16, FP16 = torch.bfloat16, torch.float16
MUTANT_CASES = lb.MUTANT_CASES


def run_case(case, mutant=None, device="cpu"):
    x = lb.make_band_inputs(case, device)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got = lm.lowp_chain(*args, mutant=mutant)
    ref = lm.oracle_chain(*args)
    model = got if mutant is None else lm.lowp_chain(*args)
    absmax = [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1], x["biases"][:c + 1])
              for c in range(len(x["ks"]))]
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)


@pytest.mark.parametrize("case", lb.BAND_SWEEP, ids=[c["id"] for c in lb.BAND_SWEEP])
def test_unmutated_model_passes(case):
    run_case(case)


def test_every_mutant_has_cases():
    assert set(MUTANT_CASES) == set(lb.BAND_MUTANTS)
    for ids in MUTANT_CASES.values():
        assert {_BY_ID[i]["dtype"] for i in ids} == {BF16, FP16}


@pytest.mark.parametrize("mutant,case_id", [(m, i) for m in lb.BAND_MUTANTS for i in MUTANT_CASES[m]],
                         ids=[f"{m}-{'bf16' if 'bf16' in i else 'fp16'}" for m in lb.BAND_MUTANTS
                              for i in MUTANT_CASES[m]])
def test_mutant_is_rejected(mutant, case_id):
    with pytest.raises(AssertionError):
        run_case(_BY_ID[case_id], mutant)


# every class of lowp_band.band_tile_classes the sweep must reach
WANT = (
    # forward: the lower edge's phase in a 128-key tile, for lo of both signs; band widths
    {("fwd_lo_phase", p, s) for p in (127, 0, 1) for s in ("neg", "pos")}
    | {("width", w) for w in (1, 63, 64, 65, 127, 128, 129, "open")}
    # forward CTA structure
    | {("wg1_later_tile",), ("wg0_ends_earlier",), ("cta_no_tile", "fresh"), ("cta_no_tile", "carried"),
       ("below_edge", "fresh"), ("below_edge", "carried")}
    # backward: i_end, need_lo, both masks on one pair, key blocks without work; deterministic turn counters
    | {("q_last", 0), ("q_last", 63), ("need_lo", 0), ("need_lo", 1), ("causal_and_lo",), ("idle_around_work",)}
    | {("det_x_min", G, kind) for G in (2, 4) for kind in ("gqa", "mqa")}
    # the host's lower-edge clamps
    | {("host_lo", v) for v in ("1-Sq", "2-Sq", "Sk", ">Sk", "=causal")}
    # carried state, key bias
    | {("chain16",), ("revived",), ("blind_last",), ("bias_edge",), ("bias_whole_band",)}
    # shapes, dtypes, layouts
    | {("sq_mod64", 1), ("sq_mod64", 63), ("sk_mod128", 1), ("sk_mod128", 127)}
    | {("dtype", n, D) for n in ("bf16", "fp16") for D in (64, 128)}
    | {("layout", L, 2) for L in ("flash", "normal", "bstride")}
)


def test_sweep_covers_every_band_edge():
    hit = set()
    for c in lb.BAND_SWEEP:
        hit |= lb.band_tile_classes(c)
    assert not WANT - hit, f"the band sweep misses {sorted(WANT - hit, key=str)}"
