"""Packed documents (cu_seqlens) on the GPU, against the fp64 document oracle under the 16-bit error model
(``lowp_model`` with the document masks of ``lowp_doc``): the doc tile kernels on every case of the document edge sweep
(chains of launches with carried state, exact zeros where nothing is attended, bitwise-reproducible deterministic
mode), the model's document faults rejected on the same inputs, ``flash_attn_varlen_func``, and the ring at W = 2, 4
and 8 on one GPU (tests/ring_harness.py)."""
import pytest
import torch

import lowp_doc
import lowp_model as lm
import ring_harness as rh

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
MUTANT_CASES = lowp_doc.mutant_cases()


def _args(x):
    return (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])


def _absmax(x):
    return [lm.scores_absmax(x["q"], x["ks"][:c + 1], x["scale"], x["masks"][:c + 1]) for c in range(len(x["ks"]))]


def native_doc_chain(x, det_runs=2):
    """The doc kernels on one case of the document sweep, straight through NativeOps: (result dict like
    lowp_chain's, [deterministic (dq, dks, dvs)])."""
    from burst_attn.chunk_ops import NativeOps
    ops = NativeOps()
    q, do, ks, vs = x["q"], x["do"], x["ks"], x["vs"]
    B, Sq, H = q.shape[:3]
    n = len(ks)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device=DEV, dtype=torch.float32)
    o_acc = torch.empty(q.shape, device=DEV, dtype=torch.float32) if n > 1 else None

    def kw(m):
        _, lo, hi, cu, q_pos0, k_pos0, ps = m
        cu_dev = torch.tensor(cu, dtype=torch.int32, device=DEV)
        return hi is not None, 0 if hi is None else hi, dict(lower=lo, doc=(cu_dev, len(cu) - 1, q_pos0, k_pos0, ps))

    states = []
    for c, m in enumerate(x["masks"]):
        causal, off, extra = kw(m)
        ops.fwd_chunk(q, ks[c], vs[c], o_acc, lse, out, x["scale"], causal, off, c == 0, c == n - 1, 1, **extra)
        if c < n - 1:
            states.append((o_acc.clone(), lse.clone()))
    delta = torch.empty(B, H, Sq, device=DEV, dtype=torch.float32)
    ops.delta(out, do, delta, 1)

    def backward(det):
        dq = torch.zeros(q.shape, device=DEV, dtype=torch.float32)
        dks, dvs = [], []
        for c, m in enumerate(x["masks"]):
            causal, off, extra = kw(m)
            dk = torch.zeros(ks[c].shape, device=DEV, dtype=torch.float32)
            dv = torch.zeros(vs[c].shape, device=DEV, dtype=torch.float32)
            ops.bwd_chunk(do, q, ks[c], vs[c], delta, lse, dq, dk, dv, x["scale"], causal, off, 1, deterministic=det,
                          **extra)
            dks.append(dk)
            dvs.append(dv)
        return dq, dks, dvs

    dq, dks, dvs = backward(False)
    dets = [backward(True) for _ in range(det_runs)]
    torch.cuda.synchronize()
    return dict(o=out, lse=lse, states=states, dq=dq, dk=dks, dv=dvs), dets


def _check_dead(x, got, ref):
    """Rows that see no key in any chunk: O = 0, dQ = 0, lse = -inf exactly; keys no row sees: dK = dV = 0."""
    dead = torch.isinf(ref["lse"]) & (ref["lse"] < 0)
    assert torch.equal(torch.isinf(got["lse"].cpu()) & (got["lse"].cpu() < 0), dead)
    rows = dead.permute(0, 2, 1)
    assert (got["o"].cpu()[rows] == 0).all(), "O of a row that sees nothing"
    assert (got["dq"].cpu()[rows] == 0).all(), "dQ of a row that sees nothing"
    B, Sq, H = x["q"].shape[:3]
    for c, (k, m) in enumerate(zip(x["ks"], x["masks"])):
        Sk, Hkv = k.shape[1], k.shape[2]
        seen = ((~dead).unsqueeze(-1) & lm.visible(Sq, Sk, m)).any(2)
        seen = seen.view(B, Hkv, H // Hkv, Sk).any(2).permute(0, 2, 1)
        for name in ("dk", "dv"):
            assert (got[name][c].cpu()[~seen] == 0).all(), f"{name} of a key no row sees (chunk {c})"


@pytest.mark.parametrize("case", lowp_doc.DOC_SWEEP, ids=[c["id"] for c in lowp_doc.DOC_SWEEP])
def test_doc_chunks_within_model(case):
    """Every case of the document edge sweep on the kernels, a chain of launches carrying the state: the fp32 state
    after each non-last chunk, O, lse, dQ, dK and dV within the 16-bit model; rows and keys with nothing to attend
    exactly zero (lse = -inf); deterministic mode bitwise reproducible and within the model."""
    x = lowp_doc.make_doc_inputs(case, DEV)
    got, dets = native_doc_chain(x)
    model, ref = lm.lowp_chain(*_args(x)), lm.oracle_chain(*_args(x))
    lm.assert_chain_within_model(case["id"], got, ref, model, case["dtype"], _absmax(x))
    _check_dead(x, got, ref)
    (dq0, dk0, dv0), (dq1, dk1, dv1) = dets
    assert torch.equal(dq0, dq1) and all(torch.equal(a, b) for a, b in zip(dk0 + dv0, dk1 + dv1)), \
        "deterministic mode is not bitwise reproducible with documents"
    lm.assert_chain_within_model(case["id"] + " deterministic", dict(got, dq=dq0, dk=dk0, dv=dv0), ref, model,
                                 case["dtype"], _absmax(x))


@pytest.mark.parametrize("mutant,dt", [(m, i) for m in lowp_doc.DOC_MUTANTS for i in (0, 1)],
                         ids=[f"{m}-{d}" for m in lowp_doc.DOC_MUTANTS for d in ("bf16", "fp16")])
def test_doc_mutants_are_rejected(mutant, dt):
    """The comparator rejects the model with a document fault, on the kernels' inputs and device."""
    case = lowp_doc._BY_ID[MUTANT_CASES[mutant][dt]]
    x = lowp_doc.make_doc_inputs(case, DEV)
    got = lm.lowp_chain(*_args(x), mutant=mutant)
    model, ref = lm.lowp_chain(*_args(x)), lm.oracle_chain(*_args(x))
    worst = dict(lm.WORST)  # the rejected runs stay out of the report of the kernels' worst ratios
    try:
        with pytest.raises(AssertionError):
            lm.assert_chain_within_model(mutant, got, ref, model, case["dtype"], _absmax(x))
    finally:
        lm.WORST.clear()
        lm.WORST.update(worst)


def test_deterministic_doc_backward_is_bitwise_reproducible():
    """GQA 4:1, head dim 128, documents at tile phases and one spanning many tiles: two deterministic runs of the
    varlen backward agree bit for bit."""
    from burst_attn.flash_triton import flash_attn_varlen_func
    torch.manual_seed(5)
    T, H, Hkv, D = 3000, 8, 2, 128
    cu = torch.tensor([0, 127, 128, 129, 700, 701, 2049, 2050, T], dtype=torch.int32, device=DEV)
    q, do = (torch.randn(T, H, D, device=DEV, dtype=torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(T, Hkv, D, device=DEV, dtype=torch.bfloat16) for _ in range(2))
    runs = []
    for _ in range(2):
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = flash_attn_varlen_func(qq, kk, vv, cu, cu, 1348, 1348, causal=True, deterministic=True)
        runs.append([o.detach()] + list(torch.autograd.grad(o, (qq, kk, vv), do)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("causal,window", [(False, (-1, -1)), (True, (-1, -1)), (True, (100, -1)), (False, (30, 70))])
def test_flash_attn_varlen_func_within_model(causal, window, monkeypatch):
    """Random document lengths incl. zero-length ones, GQA 2:1, with and without L2 blocking of the launch plan: O,
    lse, dQ, dK and dV within the 16-bit model of the packed sequence as one launch with the document mask."""
    from burst_attn.flash_triton import flash_attn_varlen_func
    g = torch.Generator().manual_seed(11)
    lens = [0, 1, 63, 64, 65, 300, 0, 1000, 129, 7, 450]
    T = sum(lens)
    cu = [0] + torch.tensor(lens).cumsum(0).tolist()
    H, Hkv, D = 4, 2, 64
    q, do = (torch.randn(1, T, H, D, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(1, T, Hkv, D, generator=g).to(torch.bfloat16) for _ in range(2))
    masks = [rh.whole_mask(dict(causal=causal, window=window, cu=cu))]
    args = (q, [k], [v], do, D ** -0.5, masks)
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    absmax = lm.scores_absmax(q, [k], D ** -0.5, masks)
    cu_dev = torch.tensor(cu, dtype=torch.int32, device=DEV)
    for blk in (None, "512"):
        if blk:
            monkeypatch.setenv("BA_L2_BLOCK", blk)
        qq, kk, vv = (t[0].to(DEV).requires_grad_() for t in (q, k, v))
        o = flash_attn_varlen_func(qq, kk, vv, cu_dev, cu_dev, max(lens), max(lens), causal=causal, window_size=window)
        lse = o.grad_fn.saved_tensors[4].detach().cpu()  # (q, k, v, out, lse) of the [1, T, H, D] view
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do[0].to(DEV))
        got = dict(o=o[None], lse=lse, dq=dq[None], dk=dk[None], dv=dv[None])
        lm.assert_api_within_model(f"varlen causal={causal} window={window} blk={blk}",
                                   {n: t.detach().cpu() for n, t in got.items()}, ref, model, torch.bfloat16, absmax)


def _jobs():
    jobs = {}
    for world in (2, 4, 8):
        S_local = 256
        S = S_local * world

        def j(mode, cu, D=128, **kw):
            return rh.ring_job(world, mode, torch.bfloat16, D, 2, S_local, cu=cu, **kw)

        cus = [[0, S], [0, 300, 301, 301, S - 129, S], list(range(0, S, 200)) + [S],
               [0, 127, 128, 129, 255, 256, 257, 511, 512, S]]
        for mode in ("none", "zigzag", "striped"):
            for n, cu in enumerate(cus):
                jobs.setdefault(world, []).append(j(mode, cu, seed=n, D=128 if n % 2 else 64))
            jobs[world].append(j(mode, cus[1], window=(150, -1), seed=9, seq_dim=2 if mode == "none" else 1))
        jobs[world].append(j("striped", cus[2], causal=False, seed=7))
        jobs[world].append(j("zigzag", cus[3], det=True, seed=8))
        if world >= 4:
            for mode in ("none", "zigzag", "striped"):
                jobs[world].append(j(mode, cus[1], intra=2, seed=10))
    return jobs


JOBS = _jobs()


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    return rh.WorldRuns(JOBS, "native", tmp_path_factory, timeout=900)


@pytest.mark.parametrize("job", [j for w in sorted(JOBS) for j in JOBS[w]], ids=lambda j: j["id"])
def test_doc_ring_on_one_device(job, runs):
    rh.check_ring_case(job, rh.load_ring_case(job, runs.outdir(job["world"])))
