"""First-contact GPU diagnostic: runs each building-block self test and a few
forward cases, printing error statistics instead of stopping at the first
failure.  Output goes to stdout and to burst_attn_diag.log in the system's temporary directory."""
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from gpu_util import err_stats, fwd_chunks, selftest  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402

import tempfile  # noqa: E402
LOG = open(os.path.join(tempfile.gettempdir(), "burst_attn_diag.log"), "a")


def say(*a):
    s = " ".join(str(x) for x in a)
    print(s, flush=True)
    LOG.write(s + "\n")
    LOG.flush()


def run(name, fn):
    try:
        say(f"[{name}]", fn())
    except Exception as e:  # noqa: BLE001
        say(f"[{name}] EXC {type(e).__name__}: {e}")
        say(traceback.format_exc())


def bwd_stage():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_bwd as tb

    def case(B, Sq, Sk, H, causal=False, off=0, dtype=torch.bfloat16):
        def f():
            q, do = tb._mk(B, Sq, H, dtype, 1), tb._mk(B, Sq, H, dtype, 2)
            k, v = tb._mk(B, Sk, H, dtype, 3), tb._mk(B, Sk, H, dtype, 4)
            got, ref = tb.run_bwd(q, k, v, do, causal, off)
            return {n: err_stats(g, r) for n, g, r in zip(("delta", "dq", "dk", "dv"), got, ref)}
        return f
    run("bwd_128x128", case(1, 128, 128, 1))
    run("bwd_256x384", case(2, 256, 384, 2))
    run("bwd_ragged_200x333", case(1, 200, 333, 2))
    run("bwd_causal_384", case(1, 384, 384, 2, True, 0))
    run("bwd_strict_384", case(1, 384, 384, 2, True, -1))
    run("bwd_fp16_256x256", case(1, 256, 256, 2, dtype=torch.float16))

    def timing():
        from burst_attn.chunk_ops import NativeOps
        ops = NativeOps()
        S, H = 16384, 32
        q, k, v, do = (torch.randn(1, S, H, 128, device="cuda").to(torch.bfloat16) for _ in range(4))
        lse = torch.full((1, H, S), 9.0, device="cuda")
        delta = torch.zeros(1, H, S, device="cuda")
        acc = [torch.zeros(1, S, H, 128, device="cuda") for _ in range(3)]
        ops.bwd_chunk(do, q, k, v, delta, lse, acc[0], acc[1], acc[2], 128 ** -0.5, False, 0, 1)
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(3):
            ops.bwd_chunk(do, q, k, v, delta, lse, acc[0], acc[1], acc[2], 128 ** -0.5, False, 0, 1)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 3
        return dict(ms=ms, tflops=2.5 * 4 * S ** 2 * H * 128 / ms / 1e9)
    run("bwd_timing_S16k_H32", timing)


def perf_stage():
    """Kernel-only timings (CUDA events, 2 warm-up + 5 timed launches) at S=32768, H=32, bf16."""
    from burst_attn.chunk_ops import NativeOps
    ops = NativeOps()
    S, H = 32768, 32
    q, k, v, do = (torch.randn(1, S, H, 128, device="cuda").to(torch.bfloat16) for _ in range(4))
    out = torch.empty_like(q)
    lse = torch.empty(1, H, S, device="cuda")
    delta = torch.zeros(1, H, S, device="cuda")
    acc = [torch.zeros(1, S, H, 128, device="cuda") for _ in range(3)]

    def t(fn, n=5):
        for _ in range(2):
            fn()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    bm = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    ms = t(lambda: torch.matmul(a, bm), 10)
    say(f"[perf calib cublas bf16 8192^3] ms={ms:.3f} tflops={2 * 8192 ** 3 / ms / 1e9:.1f}  lib={os.environ.get('BA_LIB_PATH', 'default')}")
    del a, bm
    for causal in (False, True):
        f = lambda: ops.fwd_chunk(q, k, v, None, lse, out, 128 ** -0.5, causal, 0, True, True, 1)
        ms = t(f)
        say(f"[perf fwd causal={causal}] ms={ms:.3f} "
            f"tflops={4 * S * S * H * 128 / (2 if causal else 1) / ms / 1e9:.1f}")
    for causal in (False, True):
        f = lambda: ops.bwd_chunk(do, q, k, v, delta, lse, acc[0], acc[1], acc[2], 128 ** -0.5, causal, 0, 1)
        ms = t(f)
        say(f"[perf bwd causal={causal}] ms={ms:.3f} tflops={10 * S * S * H * 128 / (2 if causal else 1) / ms / 1e9:.1f}")


def main():
    stage = sys.argv[1] if len(sys.argv) > 1 else "all"
    say("== stage", stage, torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))
    torch.manual_seed(0)
    a = torch.randn(128, 128, device="cuda").to(torch.bfloat16)
    b = torch.randn(128, 128, device="cuda").to(torch.bfloat16)

    def t_box():
        raw = selftest(2, a, b).view(torch.bfloat16).view(128, 8, 8)
        src = a[:, :64].reshape(128, 8, 8)
        exp = torch.empty_like(raw)
        for r in range(128):
            for c in range(8):
                exp[r, c ^ (r % 8)] = src[r, c]
        return dict(equal=bool(torch.equal(raw, exp)), linear_equal=bool(torch.equal(raw, src)))
    if stage in ("all", "selftest"):
        run("tma_box", t_box)
        run("ss_kmajor", lambda: err_stats(selftest(0, a, b), a.float() @ b.float().t()))
        run("ts_pv", lambda: err_stats(selftest(1, a, b), a.float() @ b.float()))
        run("ss_mnmajor", lambda: err_stats(selftest(3, a, b), a.float().t() @ b.float()))
    # variants that would match if an assumption were wrong (diagnosis aid)
        run("ts_pv_vs_AtB", lambda: err_stats(selftest(1, a, b), a.float().t() @ b.float()))
        run("ts_pv_vs_ABt", lambda: err_stats(selftest(1, a, b), a.float() @ b.float().t()))

    def fwd_case(B, Sq, Sk, H, causal=False, dtype=torch.bfloat16, nchunks=1):
        def f():
            g = torch.Generator(device="cuda").manual_seed(Sq * 7 + Sk)
            q = torch.randn(B, Sq, H, 128, device="cuda", generator=g).to(dtype)
            ks = [torch.randn(B, Sk, H, 128, device="cuda", generator=g).to(dtype) for _ in range(nchunks)]
            vs = [torch.randn(B, Sk, H, 128, device="cuda", generator=g).to(dtype) for _ in range(nchunks)]
            out, lse = fwd_chunks(q, ks, vs, 128 ** -0.5, causal=causal)
            o_ref, lse_ref = orc.dense_attention(q.cpu(), torch.cat(ks, 1).cpu(), torch.cat(vs, 1).cpu(), causal=causal)
            return dict(o=err_stats(out, o_ref), lse=err_stats(lse, lse_ref))
        return f
    if stage == "selftest":
        return
    if stage == "bwd":
        return bwd_stage()
    if stage == "perf":
        return perf_stage()
    run("fwd_128x128", fwd_case(1, 128, 128, 1))
    run("fwd_256x256", fwd_case(1, 256, 256, 2))
    run("fwd_256x1024", fwd_case(2, 256, 1024, 2))
    run("fwd_ragged_200x333", fwd_case(1, 200, 333, 2))
    run("fwd_causal_512", fwd_case(1, 512, 512, 2, causal=True))
    run("fwd_fp16_256x512", fwd_case(1, 256, 512, 2, dtype=torch.float16))
    run("fwd_chain3_256x256", fwd_case(1, 256, 256, 2, nchunks=3))

    def timing():
        q, k, v = (torch.randn(1, 16384, 32, 128, device="cuda").to(torch.bfloat16) for _ in range(3))
        fwd_chunks(q, [k], [v], 128 ** -0.5)
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(3):
            fwd_chunks(q, [k], [v], 128 ** -0.5)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 3
        return dict(ms=ms, tflops=4 * 16384 ** 2 * 32 * 128 / ms / 1e9)
    run("fwd_timing_S16k_H32", timing)


if __name__ == "__main__":
    main()
