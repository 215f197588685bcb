"""The multi-rank harness (tests/ring_harness.py) on CPU, with the fp64 oracle as the chunk operators.

The worker of tests/test_gpu_ring_one_device.py runs here on 16-bit CPU inputs: W = 2 flat and W = 4 as 2 nodes of 2,
the three shard layouts, through the staged transport, reassembled in the parent and checked against the 16-bit error
model.  The oracle passes; each ring-level fault of ``ring_harness.FAULTS`` injected into it must be rejected.  And a
rank that hangs is terminated at the timeout.
"""
import time

import pytest
import torch

import lowp_model as lm
import ring_harness as rh

BF16, FP16 = torch.bfloat16, torch.float16

JOBS = {
    2: [rh.ring_job(2, "none", BF16, 32, 2, 24),
        rh.ring_job(2, "zigzag", FP16, 32, 4, 26),
        rh.ring_job(2, "striped", BF16, 32, 1, 24, det=True),
        rh.ring_job(2, "none", FP16, 32, 2, 24, seq_dim=2, l2=16)],
    4: [rh.ring_job(4, "none", FP16, 32, 2, 16, intra=2),
        rh.ring_job(4, "zigzag", BF16, 32, 1, 18, intra=2, dq_groups=True),
        rh.ring_job(4, "striped", BF16, 32, 4, 16, intra=2, l2=16)],
}
FAULT_JOBS = [rh.ring_job(2, "striped", BF16, 32, 2, 24, fault="striped_not_strict"),
              rh.ring_job(2, "zigzag", BF16, 32, 2, 24, fault="lost_dq_hop"),
              rh.ring_job(2, "none", FP16, 32, 2, 24, fault="fwd_state_dropped")]
JOBS[2] += FAULT_JOBS


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    return rh.WorldRuns(JOBS, "oracle", tmp_path_factory, timeout=300)


@pytest.fixture
def own_worst(monkeypatch):
    monkeypatch.setattr(lm, "WORST", {})


@pytest.mark.parametrize("job", [j for w in JOBS for j in JOBS[w] if not j["fault"]], ids=lambda j: j["id"])
def test_oracle_ring_within_model(runs, job, own_worst):
    rh.check_ring_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))


def test_every_fault_has_a_control():
    assert sorted(j["fault"] for j in FAULT_JOBS) == sorted(rh.FAULTS)


@pytest.mark.parametrize("job", FAULT_JOBS, ids=lambda j: j["fault"])
def test_ring_fault_is_rejected(runs, job, own_worst):
    got = rh.load_ring_case(job, runs.outdir(job["world"]))
    with pytest.raises(AssertionError):
        rh.check_ring_case(job, got)


def _hang_on_rank1(rank, world, port):
    if rank == 1:
        time.sleep(3600)


def test_spawn_terminates_a_hung_rank():
    t0 = time.monotonic()
    with pytest.raises(AssertionError, match=r"ranks \[1\] still running"):
        rh.spawn(_hang_on_rank1, 2, timeout=20)
    assert time.monotonic() - t0 < 45
