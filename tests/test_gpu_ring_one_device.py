"""The ring at W = 2, 4 and 8 with the native kernels, on one GPU, against the 16-bit error model.

W ranks run as W processes that all use cuda:0 under one gloo process group (tests/ring_harness.py).  Every chunk
operation is the real ``NativeOps``: the tile kernels get the zigzag half views, the causal offsets of striped rounds,
the fp32 state carried across rounds, the dQ partials reduce-added on arrival, GQA dK/dV summed across rounds and the
L2-blocked sub-launches exactly as the ring driver passes them.  Only the hop is replaced: it is staged through the
CPU, with NaN in every receive buffer and a snapshot check of every source while the hop is in flight, so a kernel
that reads a buffer too early or writes one too soon fails.  The NCCL and copy-engine transports are covered by
tests/test_gpu_ring_multi.py on two or more GPUs.

Per case the parent reassembles O, lse, dQ, dK and dV of the full sequence and checks them against the fp64 oracle
and the 16-bit model of the whole sequence as one chunk (``lowp_model.assert_api_within_model``); each rank checks
that the caller's q, k, v are unchanged, and deterministic cases run twice and must be bitwise equal.  Three ring-level
faults injected into the native operators (``ring_harness.FAULTS``) must be rejected.
"""
import ctypes
import ctypes.util

import pytest
import torch

pytestmark = pytest.mark.gpu

import lowp_model as lm  # noqa: E402
import ring_harness as rh  # noqa: E402

BF16, FP16 = torch.bfloat16, torch.float16


def _flat_cases(world, B):
    j = lambda *a, **kw: rh.ring_job(world, *a, B=B, **kw)  # noqa: E731
    return [j("none", BF16, 128, 4, 256), j("zigzag", BF16, 128, 4, 256), j("striped", BF16, 128, 4, 256),
            j("none", FP16, 64, 2, 130),
            j("zigzag", FP16, 64, 2, 130),                   # halves of 65 rows
            j("striped", FP16, 64, 1, 130),
            j("zigzag", BF16, 80, 1, 258, scale=0.3),        # head_dim padded to 128; halves of 129 rows
            j("none", BF16, 128, 2, 258, seq_dim=2),         # [B,H,S,D] (flash=None)
            j("zigzag", BF16, 128, 2, 320, l2=128, det=True),
            j("striped", FP16, 128, 4, 320, l2=128, det=True)]


JOBS = {
    2: _flat_cases(2, 2),
    4: _flat_cases(4, 2) + [
        rh.ring_job(4, "none", BF16, 128, 2, 256, intra=2, dq_groups=True),
        rh.ring_job(4, "zigzag", FP16, 64, 4, 130, intra=2, dq_groups=True),
        rh.ring_job(4, "striped", BF16, 128, 1, 258, intra=2, dq_groups=True, det=True)],
    8: [rh.ring_job(8, m, BF16, 128, 2, 128, B=1) for m in ("none", "zigzag", "striped")] + [
        rh.ring_job(8, "zigzag", FP16, 64, 4, 130, B=1)] + [
        rh.ring_job(8, m, BF16, 128, 2, 128, B=1, intra=intra, dq_groups=intra == 4)
        for intra in (4, 2) for m in ("zigzag", "striped")],
}
# negative controls: one matching case each, at W = 4 without L2 blocking
FAULT_JOBS = [rh.ring_job(4, "striped", BF16, 128, 4, 256, fault="striped_not_strict"),
              rh.ring_job(4, "zigzag", BF16, 128, 4, 256, fault="lost_dq_hop"),
              rh.ring_job(4, "none", BF16, 128, 4, 256, fault="fwd_state_dropped")]
JOBS[4] += FAULT_JOBS
CASES = [j for w in JOBS for j in JOBS[w] if not j["fault"]]
for _j in CASES + FAULT_JOBS:  # oracle_chain holds several [B,H,S,S] fp64 tensors
    assert _j["case"]["B"] * 4 * _j["case"]["sq"] ** 2 <= 2 * 4 * 2048 ** 2, _j["id"]

RING_WORST: dict = {}  # lm.WORST of the ring cases only


def _compute_mode():
    """The device's compute mode, read-only through the driver API (0: default, 2: prohibited, 3: exclusive
    process); None when it cannot be read."""
    name = ctypes.util.find_library("cuda") or "libcuda.so.1"
    try:
        cu = ctypes.CDLL(name)
    except OSError:
        return None
    dev, mode = ctypes.c_int(), ctypes.c_int()
    if cu.cuInit(0) or cu.cuDeviceGet(ctypes.byref(dev), 0):
        return None
    if cu.cuDeviceGetAttribute(ctypes.byref(mode), 20, dev):  # CU_DEVICE_ATTRIBUTE_COMPUTE_MODE
        return None
    return mode.value


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) != (9, 0):
        pytest.skip("needs an sm_90 GPU")
    mode = _compute_mode()
    if mode != 0:
        pytest.skip(f"W ranks share cuda:0, which needs the Default compute mode (read {mode})")
    return rh.WorldRuns(JOBS, "native", tmp_path_factory, timeout=900)


@pytest.fixture
def ring_worst(monkeypatch):
    monkeypatch.setattr(lm, "WORST", RING_WORST)


@pytest.mark.parametrize("job", CASES, ids=lambda j: j["id"])
def test_ring_within_model(runs, job, ring_worst):
    rh.check_ring_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))


@pytest.mark.parametrize("job", FAULT_JOBS, ids=lambda j: j["fault"])
def test_ring_fault_is_rejected(runs, job, monkeypatch):
    monkeypatch.setattr(lm, "WORST", {})
    got = rh.load_ring_case(job, runs.outdir(job["world"]))
    with pytest.raises(AssertionError) as e:
        rh.check_ring_case(job, got)
    print(f"\n{job['fault']}: {str(e.value)[:160]}")


def test_report_worst_ratios():
    """Runs last: prints the worst error / bound of the ring cases per output and dtype."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(RING_WORST.items()):
        print(f"worst ring {name:>4s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
