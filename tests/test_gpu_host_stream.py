"""Host-resident operands (burst_attn/host_stream.py): burst_attn_func called with pinned CPU tensors on one rank
streams Q/K/V/dO up on an upload stream and O/dQ/dK/dV down on a download stream, under the L2-blocked sub-launches
on the compute stream.

* A sweep of calls (bf16 / fp16, head dims 64 and 128, B = 1 and 2, the [B,S,H,D] and [B,H,S,D] layouts, MHA, GQA
  2:1 and 4:1, MQA, causal and not, L2 blocks of one block, blocks that divide S, a ragged last block, blocks that are
  not a multiple of the 128-row tile and one-row / one-key last blocks): O, lse, dQ, dK and dV within the 16-bit error
  model (``lowp_model``) of the whole call as one chunk, and close to the same call on device tensors; with
  deterministic=True two calls are bitwise equal.
* Ordering: a busy-wait kernel (``torch.cuda._sleep``) delays the upload, download or compute stream just before the
  forward or the backward, while every device buffer the module allocates and every pinned buffer it returns starts as
  NaN.  After a synchronize the results are bitwise those of the undelayed call: a kernel that missed a wait, or a
  download that started before its cast, reads NaN or stale memory.
* Autograd consumers read the host gradients the moment the backward returns: gradient accumulation (``q.grad +=``)
  and tensor hooks, with the download stream delayed.
* Unsupported options are rejected before any copy or launch.
"""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

import lowp_model as lm  # noqa: E402
from burst_attn import burst_attn_func, burst_attn_func_striped, host_stream  # noqa: E402

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
GRADS = ("dq", "dk", "dv")
OUTPUTS = ("o", "lse") + GRADS
SLEEP_CYCLES = 250_000_000  # SM clock cycles of torch.cuda._sleep: 0.13 s at 1980 MHz, 0.18 s at 1400 MHz
HOST_WORST: dict = {}


def _case(S, blk, causal, dtype=torch.bfloat16, D=128, B=1, H=3, Hkv=None, layout="flash", det=False, seed=0):
    Hkv = Hkv or H
    name = (f"S{S}_blk{blk}_{'causal' if causal else 'full'}_{'bf16' if dtype == torch.bfloat16 else 'fp16'}_d{D}"
            f"_B{B}H{H}kv{Hkv}_{layout}" + ("_det" if det else ""))
    assert layout == "flash" or not causal, "causal attention needs flash='cuda'"
    return dict(id=name, S=S, blk=blk, causal=causal, dtype=dtype, D=D, B=B, H=H, Hkv=Hkv, layout=layout, det=det,
                seed=seed, scale=D ** -0.5)


BF, FP = torch.bfloat16, torch.float16
CASES = [
    # one block (S < block), blocks that divide S, a ragged last block
    *[_case(S, blk, c) for S, blk in ((1024, 256), (1536 + 200, 512), (384, 32768)) for c in (False, True)],
    # blocks that are not a multiple of the 128-row tile
    _case(1000, 200, False, FP, 64),
    _case(1000, 200, True, FP, 64, det=True),
    # one-row / one-key last blocks, B = 2 (every copy of a block is strided)
    _case(257, 128, True, BF, 64, B=2, H=2, det=True),
    _case(129, 128, True, FP, 128, B=2, H=4, Hkv=2),
    # [B,H,S,D]: every block of every head is a strided copy
    _case(257, 128, False, FP, 128, B=2, H=2, layout="normal", det=True),
    _case(1000, 200, False, BF, 128, B=2, H=4, Hkv=2, layout="normal"),
    _case(200, 512, False, FP, 64, B=2, H=4, Hkv=1, layout="normal"),
    # GQA 4:1 (Hq = 8, Hkv = 2) and MQA (Hkv = 1)
    _case(1024 + 100, 256, False, BF, 128, H=8, Hkv=2),
    _case(1024 + 100, 256, True, BF, 128, H=8, Hkv=2, det=True),
    _case(700, 256, True, FP, 64, B=2, H=4, Hkv=1, det=True),
]
# the ordering checks: one call whose copies are all asynchronous (B = 1, [B,S,H,D]), one whose are all strided
ORDER_CASES = [_case(1000, 256, True, BF, 128, seed=1),
               _case(600, 256, False, FP, 64, B=2, H=4, Hkv=2, layout="normal", seed=2)]


def _operands(case):
    """dict(flash: the logical [B,S,H,D] CPU tensors q, k, v, do; call: the same, pinned, in the call's layout)."""
    g = torch.Generator().manual_seed(case["seed"])
    B, S, H, Hkv, D, dt = (case[n] for n in ("B", "S", "H", "Hkv", "D", "dtype"))
    q, do = (torch.randn(B, S, H, D, generator=g).to(dt) for _ in range(2))
    k, v = (torch.randn(B, S, Hkv, D, generator=g).to(dt) for _ in range(2))
    flash = dict(q=q, k=k, v=v, do=do)
    lay = (lambda t: t) if case["layout"] == "flash" else (lambda t: t.transpose(1, 2).contiguous())
    return dict(flash=flash, call={n: lay(t).pin_memory() for n, t in flash.items()})


def _stream(name):
    up, down = host_stream._copy_streams(DEV)
    return {"up": up, "down": down, "compute": torch.cuda.current_stream(DEV)}[name]


def _sleep_on(name):
    with torch.cuda.stream(_stream(name)):
        torch.cuda._sleep(SLEEP_CYCLES)


def _host_call(case, x, deterministic, delay=None):
    """burst_attn_func on the pinned operands ``x["call"]`` and its backward through autograd.  ``delay``: (stream,
    "fwd" | "bwd"), a busy-wait on that stream just before that half.  Returns the outputs in the call's layout (lse
    [B,H,S]) and the wall time from the forward to the end of a device synchronize."""
    t0 = time.perf_counter()
    q, k, v = (x["call"][n].detach().requires_grad_() for n in "qkv")
    if delay and delay[1] == "fwd":
        _sleep_on(delay[0])
    o = burst_attn_func(q, k, v, case["scale"], "cuda" if case["layout"] == "flash" else None, case["causal"], False,
                        deterministic)
    lse = o.grad_fn.saved_tensors[4]  # host_stream.forward saves (qd, kd, vd, out, lse)
    if delay and delay[1] == "bwd":
        _sleep_on(delay[0])
    dq, dk, dv = torch.autograd.grad(o, (q, k, v), x["call"]["do"])
    torch.cuda.synchronize()
    return dict(o=o.detach(), lse=lse.cpu(), dq=dq, dk=dk, dv=dv, seconds=time.perf_counter() - t0)


def _flash(case, t):
    return t if case["layout"] == "flash" else t.transpose(1, 2)


def _check_within_model(case, x, got, name):
    f = {n: t.to(DEV) for n, t in x["flash"].items()}
    mask = ("causal_offset", 0) if case["causal"] else None
    args = (f["q"], [f["k"]], [f["v"]], f["do"], case["scale"], [mask])
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args, device=DEV)
    absmax = lm.scores_absmax(f["q"], [f["k"]], case["scale"], [mask], device=DEV)
    res = {n: got[n] if n == "lse" else _flash(case, got[n]) for n in OUTPUTS}
    lm.assert_api_within_model(name, res, ref, model, case["dtype"], absmax)


@pytest.fixture
def host_worst(monkeypatch):
    monkeypatch.setattr(lm, "WORST", HOST_WORST)


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_host_resident_call_matches_oracle_and_device_call(monkeypatch, host_worst, case):
    monkeypatch.setenv("BA_L2_BLOCK", str(case["blk"]))
    x = _operands(case)
    runs = [_host_call(case, x, case["det"]) for _ in range(2 if case["det"] else 1)]
    got = runs[0]
    for n in ("o", "dq"):
        assert got[n].device.type == "cpu" and got[n].dtype == case["dtype"] and got[n].shape == x["call"]["q"].shape
    for n in ("dk", "dv"):
        assert got[n].device.type == "cpu" and got[n].dtype == case["dtype"] and got[n].shape == x["call"]["k"].shape
    _check_within_model(case, x, got, case["id"])
    if case["det"]:
        for n in OUTPUTS:
            assert torch.equal(runs[0][n], runs[1][n]), f"{n}: two deterministic host-resident calls differ"
    # and the plain device call on the same inputs (zigzag shards need an even S; at W = 1 the striped call is plain
    # causal attention as well)
    fn = burst_attn_func_striped if case["causal"] and case["S"] % 2 else burst_attn_func
    qd, kd, vd = (x["call"][n].to(DEV).requires_grad_() for n in "qkv")
    od = fn(qd, kd, vd, case["scale"], "cuda" if case["layout"] == "flash" else None, case["causal"],
                         False, case["det"])
    gd = torch.autograd.grad(od, (qd, kd, vd), x["call"]["do"].to(DEV))
    for n, ref in zip(("o",) + GRADS, (od, *gd)):
        torch.testing.assert_close(got[n].float(), ref.float().cpu(), rtol=2e-2, atol=2e-2, msg=n)


class _NanTorch:
    """``torch`` as host_stream sees it in the ordering checks: ``empty`` / ``empty_like`` are NaN-filled (on the
    stream that allocates them), so whatever reads a buffer before its copy or kernel has written it reads NaN, not
    a previous call's values that the caching allocator happens to hand back."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def empty(*a, **k):
        return _nan(torch.empty(*a, **k))

    @staticmethod
    def empty_like(t, **k):
        return _nan(torch.empty_like(t, **k))


def _nan(t):
    assert t.is_floating_point(), t.dtype
    return t.fill_(float("nan"))


def _poison(monkeypatch):
    monkeypatch.setattr(host_stream, "torch", _NanTorch())
    monkeypatch.setattr(host_stream, "_pinned_like",
                        lambda shape, dtype: _nan(torch.empty(shape, dtype=dtype, pin_memory=True)))


@pytest.fixture(scope="module")
def sleep_seconds():
    """How long one delay busy-waits, by CUDA events (the second of two, after the kernel's module is loaded)."""
    for _ in range(2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.cuda._sleep(SLEEP_CYCLES)
        b.record()
        b.synchronize()
    return a.elapsed_time(b) / 1e3


@pytest.mark.parametrize("phase", ["fwd", "bwd"])
@pytest.mark.parametrize("stream", ["up", "down", "compute"])
@pytest.mark.parametrize("case", ORDER_CASES, ids=[c["id"] for c in ORDER_CASES])
def test_delayed_stream_and_nan_buffers_leave_results_bitwise_unchanged(monkeypatch, sleep_seconds, case, stream,
                                                                        phase):
    """Delay one stream before one half of the call, with NaN in every buffer host_stream allocates: after a
    synchronize O, lse, dQ, dK and dV are bitwise those of the undelayed call (deterministic=True), and the delay did
    hold the call up."""
    monkeypatch.setenv("BA_L2_BLOCK", str(case["blk"]))
    x = _operands(case)
    _host_call(case, x, True)  # the pinned and device blocks the two calls below reuse
    ref = _host_call(case, x, True)
    _poison(monkeypatch)
    got = _host_call(case, x, True, delay=(stream, phase))
    for n in OUTPUTS:
        assert not torch.isnan(got[n]).any(), f"{n}: NaN with the {stream} stream delayed before the {phase}"
        assert torch.equal(got[n], ref[n]), f"{n}: differs with the {stream} stream delayed before the {phase}"
    lag = got["seconds"] - ref["seconds"]
    print(f"\n{case['id']} {stream} before {phase}: {ref['seconds'] * 1e3:.1f} ms undelayed, "
          f"{got['seconds'] * 1e3:.1f} ms delayed, sleep {sleep_seconds * 1e3:.1f} ms")
    assert lag > 0.5 * sleep_seconds, f"the {stream} delay held the call up by {lag * 1e3:.1f} ms only"


def _undelayed_grads(monkeypatch, case, x):
    monkeypatch.setenv("BA_L2_BLOCK", str(case["blk"]))
    ref = _host_call(case, x, True)
    return [ref[n] for n in GRADS]


def test_gradient_accumulation_sums_finished_host_gradients(monkeypatch):
    """Two backward passes into the same pinned leaves, the download stream delayed before each: AccumulateGrad adds
    the second gradient to the first on the host as soon as the backward returns, so q.grad (k, v) must be the bf16
    sum of two undelayed gradients, bitwise."""
    case = ORDER_CASES[0]
    x = _operands(case)
    want = [g + g for g in _undelayed_grads(monkeypatch, case, x)]
    _poison(monkeypatch)
    leaves = [x["call"][n].detach().requires_grad_() for n in "qkv"]
    o = burst_attn_func(*leaves, case["scale"], "cuda", case["causal"], False, True)
    for i in range(2):
        _sleep_on("down")
        o.backward(x["call"]["do"], retain_graph=i == 0)
    torch.cuda.synchronize()
    for n, t, w in zip(GRADS, leaves, want):
        assert not torch.isnan(t.grad).any(), f"{n}: accumulated gradient holds NaN"
        assert torch.equal(t.grad, w), f"{n}: accumulated gradient is not the sum of two finished gradients"


def test_tensor_hooks_see_finished_host_gradients(monkeypatch):
    """Hooks on the pinned leaves clone their gradient the moment autograd passes it on, with the download stream
    delayed before the backward: the clones are the undelayed gradients, bitwise."""
    case = ORDER_CASES[0]
    x = _operands(case)
    want = _undelayed_grads(monkeypatch, case, x)
    _poison(monkeypatch)
    leaves = [x["call"][n].detach().requires_grad_() for n in "qkv"]
    seen = {}

    def hook(n):
        def save(g):
            seen[n] = g.clone()
        return save

    for n, t in zip(GRADS, leaves):
        t.register_hook(hook(n))
    o = burst_attn_func(*leaves, case["scale"], "cuda", case["causal"], False, True)
    _sleep_on("down")
    o.backward(x["call"]["do"])
    torch.cuda.synchronize()
    for n, w in zip(GRADS, want):
        assert not torch.isnan(seen[n]).any(), f"{n}: the hook saw NaN"
        assert torch.equal(seen[n], w), f"{n}: the hook saw an unfinished gradient"


REJECTED = {"window_size": (NotImplementedError, "window_size is not supported with host-resident"),
            "alibi_slopes": (NotImplementedError, "alibi_slopes is not supported with host-resident"),
            "cu_seqlens": (NotImplementedError, "cu_seqlens is not supported with host-resident"),
            "head_dim": (AssertionError, "head_dim 64 or 128")}


@pytest.mark.parametrize("what", sorted(REJECTED))
def test_unsupported_host_calls_are_rejected_before_any_copy(monkeypatch, what):
    """window_size, alibi_slopes and cu_seqlens raise NotImplementedError, a head dim other than 64 or 128 fails its
    assertion, all before host_stream.forward copies or launches anything."""
    def copies(*a, **k):
        pytest.fail(f"{what}: host_stream.forward ran before the call was rejected")

    monkeypatch.setattr(host_stream, "forward", copies)
    S, H = 256, 2
    D = 96 if what == "head_dim" else 64
    q, k, v = (torch.randn(1, S, H, D).to(torch.bfloat16).pin_memory().requires_grad_() for _ in range(3))
    kw = dict(window_size=dict(window_size=(32, 32)), alibi_slopes=dict(alibi_slopes=torch.full((H,), 0.25)),
              cu_seqlens=dict(cu_seqlens=torch.tensor([0, 100, S], dtype=torch.int32))).get(what, {})
    exc, match = REJECTED[what]
    with pytest.raises(exc, match=match):
        burst_attn_func(q, k, v, None, "cuda", False, **kw)


def test_cpu_tensors_without_pinning_fail_loudly():
    q = torch.randn(1, 128, 1, 128, dtype=torch.bfloat16)
    with pytest.raises(AssertionError):
        burst_attn_func(q, q, q, None, "cuda", False)


def test_report_worst_ratios():
    """Runs last: prints the worst error / bound of the host-resident calls per output and dtype."""
    for (name, dt), ((g, gcase), (r, rcase)) in sorted(HOST_WORST.items()):
        print(f"worst host {name:>4s} {dt:>8s}: global {g:6.3f} ({gcase})  row {r:6.3f} ({rcase})")
