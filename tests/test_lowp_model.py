"""The 16-bit error model and its comparator (tests/lowp_model.py), without a GPU.

* Unmutated: the model, standing in for the kernels, passes the comparator against the fp64 oracle on every case of
  the tile-edge sweep (tests/test_gpu_tile_edges.py runs the same cases on the kernels).
* Mutants: each realistic kernel fault of ``lowp_model.MUTANTS``, injected into the model, is rejected -- on a
  bf16 and on an fp16 case.  A mutant that passes means the comparator is too loose.
"""
import pytest
import torch

import lowp_model as lm

_BY_ID = {c["id"]: c for c in lm.SWEEP}


def _run(case, mutant=None):
    x = lm.make_inputs(case)
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    got = lm.lowp_chain(*args, mutant=mutant)
    ref = lm.oracle_chain(*args)
    model = got if mutant is None else lm.lowp_chain(*args)
    n = len(x["ks"])
    absmax = [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1], x["biases"][:c + 1])
              for c in range(n)]
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], absmax)


@pytest.mark.parametrize("case", lm.SWEEP, ids=[c["id"] for c in lm.SWEEP])
def test_unmutated_model_passes(case):
    _run(case)


# per mutant: one bf16 and one fp16 case of the sweep on which the fault is live
_MUTANT_CASES = {
    "drop_key_127": ["q128_k257_d128_bf16_sd_randn", "q128_k257_d64_fp16_sd_randn"],
    "drop_key_128": ["q128_k257_d128_bf16_sd_randn", "q128_k257_d64_fp16_sd_randn"],
    "drop_key_last": ["q257_k513_d128_bf16_sd_randn", "q65_k127_d64_fp16_sd_randn"],
    "causal_plus1_fwd": ["q255_k257@1_d128_bf16_sd_randn", "q255_k257@0_d128_fp16_sd_randn"],
    "causal_minus1_fwd": ["q255_k257@1_d128_bf16_sd_randn", "q255_k257@0_d128_fp16_sd_randn"],
    "causal_plus1_bwd": ["q255_k257@1_d128_bf16_sd_randn", "q255_k257@0_d128_fp16_sd_randn"],
    "causal_minus1_bwd": ["q255_k257@1_d128_bf16_sd_randn", "q255_k257@0_d128_fp16_sd_randn"],
    "strict_swap": ["q129_k513@127_d128_bf16_sd_randn", "q129_k129@0_d64_fp16_sd_randn"],
    "scale_fwd": ["q129_k257_d128_bf16_s0.3_last_tile", "q129_k257_d128_fp16_s0.3_randn"],
    "scale_bwd": ["q129_k257@128_d64_bf16_s1.0_randn", "q129_k257@128_d64_fp16_s1.0_last_tile"],
    "bias_natural_fwd": ["q129_k257_d128_bf16_sd_randn_bias-randn", "q129_k257_d64_fp16_sd_randn_bias-randn"],
    "bias_natural_bwd": ["q129_k257_d128_bf16_sd_randn_bias-randn", "q129_k257_d64_fp16_sd_randn_bias-randn"],
    "carried_l4": ["q129_k128+129_d128_bf16_sd_randn", "q129_k128+129_d64_fp16_sd_randn"],
    "dead_revive_stale_m": ["dead1st_q129_k128@-129+128@128+129@0_d128_bf16_sd_randn",
                            "dead1st_q129_k128@-129+128@128+129@0_d64_fp16_sd_randn"],
    "gqa_wrong_head": ["q129_k257@127_d64_bf16_sd_randn_B1H4kv2", "q129_k257@127_d128_fp16_sd_randn_B1H4kv2"],
    "dk_no_scale": ["q257_k513_d128_bf16_sd_randn", "q257_k513_d64_fp16_sd_randn"],
    "dq_missing_key_block": ["q257_k513_d128_bf16_sd_randn", "q257_k513_d64_fp16_sd_randn"],
    "dv_missing_q_block": ["q255_k257@1_d128_bf16_sd_randn", "q255_k257@0_d128_fp16_sd_randn"],
}


def test_every_mutant_has_cases():
    assert set(_MUTANT_CASES) == set(lm.MUTANTS)
    for ids in _MUTANT_CASES.values():
        assert {_BY_ID[i]["dtype"] for i in ids} == {torch.bfloat16, torch.float16}


@pytest.mark.parametrize("mutant,case_id", [(m, i) for m in lm.MUTANTS for i in _MUTANT_CASES[m]],
                         ids=[f"{m}-{'bf16' if 'bf16' in i else 'fp16'}" for m in lm.MUTANTS for i in _MUTANT_CASES[m]])
def test_mutant_is_rejected(mutant, case_id):
    with pytest.raises(AssertionError):
        _run(_BY_ID[case_id], mutant)
