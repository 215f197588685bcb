"""A/B of two builds of libburst_attn_b200.so on the flagship benchmark: fresh processes, alternating.

    python tools/ab_lib.py --build-base REV      build REV's library (git archive + make) into build/ab/base/
    python tools/ab_lib.py [--rounds 5] [--seq 65536] [--steps 5] [--warmup 3] [--check-outputs DIR] [--out FILE]

bench.py loads the library once per process, so every timed run is a fresh `bench.py --gpus 1 --no-cpu --no-e2e`
with BA_LIB_PATH set to one of the two libraries, in the order base, new, base, new, ... (R runs each).  Default
libraries: build/ab/base/libburst_attn_b200.so (made by --build-base; build/ is git-ignored but is part of the working
tree) against the in-tree build burst-attention_b200/lib/libburst_attn_b200.so.  The card name, power limit and
maximum SM clock are read once in the same call; each run's SM clock is the median bench.py sampled while it timed.

Printed per variant: median / min / max of value (fwd+bwd TFLOPS/s), ms_per_step, fwd_tflops, roofline.achieved
(the backward kernel's TFLOP/s), roofline.fwd_kernel.achieved and clocks.sm_mhz, then one JSON line with all runs.

--check-outputs DIR compares what the two libraries compute on the same seeded inputs, before the timed runs:
  * bench.py --steps 2 --dump-outputs (same seed, --seq): O, dK, dV must be bitwise equal; dQ, whose fp32 reduce-add
    order across key blocks is unordered, is reported as its largest difference (absolute and in bf16 steps) next
    to the difference between two runs of the base library;
  * dQ of one deterministic-mode backward chunk (Sq = Sk = 4096, H = 32, D = 128, bf16) must be bitwise equal.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_DIR = os.path.join(ROOT, "build", "ab", "base")
LIB_NAME = "libburst_attn_b200.so"
FIELDS = (("value", ("value",)), ("ms_per_step", ("ms_per_step",)), ("fwd_tflops", ("fwd_tflops",)),
          ("bwd_kernel_tflops", ("roofline", "achieved")), ("fwd_kernel_tflops", ("roofline", "fwd_kernel", "achieved")),
          ("sm_mhz", ("clocks", "sm_mhz")))


def build_base(rev):
    """Export `rev` from git into a temporary directory, build its libraries there, copy them to build/ab/base/."""
    sha = subprocess.run(["git", "-C", ROOT, "rev-parse", rev], capture_output=True, text=True, check=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        tar_path = os.path.join(tmp, "src.tar")
        with open(tar_path, "wb") as f:
            subprocess.run(["git", "-C", ROOT, "archive", sha], stdout=f, check=True)
        src = os.path.join(tmp, "src")
        with tarfile.open(tar_path) as t:
            t.extractall(src, filter="data")
        res = subprocess.run(["make", "-C", os.path.join(src, "burst-attention_b200", "csrc"), "-j8"],
                             capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise SystemExit(f"building {rev} ({sha}) failed")
        os.makedirs(BASE_DIR, exist_ok=True)
        lib_dir = os.path.join(src, "burst-attention_b200", "lib")
        for name in os.listdir(lib_dir):
            shutil.copy2(os.path.join(lib_dir, name), os.path.join(BASE_DIR, name))
    with open(os.path.join(BASE_DIR, "REVISION"), "w") as f:
        f.write(sha + "\n")
    print(f"built {rev} ({sha}) -> {BASE_DIR}")


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, smax = (x.strip() for x in out.split(","))
        return {"card": name, "power_limit_w": float(plim), "sm_max_mhz": int(float(smax))}
    except Exception as e:  # noqa: BLE001
        return {"nvidia_smi": f"unavailable ({type(e).__name__})"}


def run_bench(lib, extra):
    env = dict(os.environ, BA_LIB_PATH=lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu", "--no-e2e", *extra]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise SystemExit(f"bench.py failed with BA_LIB_PATH={lib} (exit {res.returncode})")
    return json.loads(lines[-1])


def pick(d, path):
    for k in path:
        d = d.get(k) if isinstance(d, dict) else None
    return d


def det_dq(out_path):
    """Child process: dQ of one deterministic backward chunk with the library BA_LIB_PATH names -> out_path (.npy)."""
    import numpy as np
    import torch
    sys.path[:0] = [ROOT, os.path.join(ROOT, "burst-attention_b200")]
    from burst_attn.chunk_ops import NativeOps
    from oracle import attention_oracle as orc
    S, H, D = 4096, 32, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    q, k, v, do = (torch.randn(1, S, H, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    scale = D ** -0.5
    o, lse = orc.dense_attention(q, k, v, scale, False, torch.float32)
    delta = orc.compute_delta(o, do, torch.float32)
    acc = [torch.zeros(t.shape, device="cuda", dtype=torch.float32) for t in (q, k, v)]
    NativeOps().bwd_chunk(do, q, k, v, delta, lse.contiguous(), acc[0], acc[1], acc[2], scale, False, 0, 1,
                          deterministic=True)
    torch.cuda.synchronize()
    np.save(out_path, acc[0].cpu().numpy())


def bf16_ulps(a, b):
    """Largest distance in bf16 steps between two float32 arrays that hold bf16 values."""
    import numpy as np

    def ordinal(x):
        bits = (x.astype(np.float32).view(np.int32) >> 16).astype(np.int64)
        return np.where(bits < 0, -(bits & 0x7FFF), bits)
    return int(np.abs(ordinal(a) - ordinal(b)).max()) if a.size else 0


def check_outputs(libs, out_dir, seq):
    """O, dK, dV and the deterministic dQ must be bitwise equal.  The default dQ adds the key blocks' partials in
    whatever order their reduce-adds reach L2, so it differs between any two runs, even of one library: its
    difference new vs base is reported next to that of a second base run against the first."""
    import numpy as np
    report = {}
    for name, lib in (*libs.items(), ("base2", libs["base"])):
        run_bench(lib, ["--steps", "2", "--seq", str(seq), "--dump-outputs", os.path.join(out_dir, name)])
        if name == "base2":
            continue
        res = subprocess.run([sys.executable, __file__, "--det-dq", os.path.join(out_dir, f"det_dq_{name}.npy")],
                             env=dict(os.environ, BA_LIB_PATH=lib), capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
            raise SystemExit(f"deterministic dQ run failed with BA_LIB_PATH={lib}")
    ld = lambda *p: np.load(os.path.join(out_dir, *p))  # noqa: E731

    def diff(a, b):
        return {"bitwise_equal": bool(np.array_equal(a, b)), "max_abs_diff": float(np.abs(a - b).max()),
                "max_bf16_ulps": bf16_ulps(a, b), "n_differ": int((a != b).sum()), "n": int(a.size)}
    for t in ("o", "dk", "dv", "dq"):
        report[t] = diff(ld("base", f"{t}.npy"), ld("new", f"{t}.npy"))
    report["dq_base_vs_base"] = diff(ld("base", "dq.npy"), ld("base2", "dq.npy"))
    report["deterministic_dq"] = diff(ld("det_dq_base.npy"), ld("det_dq_new.npy"))
    ok = all(report[t]["bitwise_equal"] for t in ("o", "dk", "dv", "deterministic_dq"))
    report["ok"] = ok
    print(json.dumps({"check_outputs": report}), flush=True)
    return ok


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--build-base", metavar="REV", help="build REV's library into build/ab/base/ and exit")
    ap.add_argument("--base", default=os.path.join(BASE_DIR, LIB_NAME))
    ap.add_argument("--new", default=os.path.join(ROOT, "burst-attention_b200", "lib", LIB_NAME))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seq", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check-outputs", metavar="DIR", help="compare the two libraries' outputs first (see above)")
    ap.add_argument("--out", help="also write the JSON summary to this file")
    ap.add_argument("--det-dq", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.build_base:
        return build_base(args.build_base)
    if args.det_dq:
        return det_dq(args.det_dq)
    libs = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    for name, lib in libs.items():
        if not os.path.exists(lib):
            raise SystemExit(f"{name} library {lib} is missing (tools/ab_lib.py --build-base REV makes the base)")

    checked = check_outputs(libs, args.check_outputs, args.seq) if args.check_outputs else None
    runs = {name: [] for name in libs}
    for r in range(args.rounds):
        for name, lib in libs.items():
            line = run_bench(lib, ["--seq", str(args.seq), "--steps", str(args.steps), "--warmup", str(args.warmup)])
            row = {f: pick(line, path) for f, path in FIELDS}
            runs[name].append(row)
            print(f"round {r} {name:4s} " + " ".join(f"{f}={row[f]:.1f}" if isinstance(row[f], (int, float))
                                                    else f"{f}={row[f]}" for f in row), flush=True)
    info = device_info()
    print(f"\n{info}  S={args.seq} steps={args.steps} warmup={args.warmup} rounds={args.rounds}")
    print(f"{'field':>18s} | " + " | ".join(f"{n:>26s}" for n in libs))
    summary = {}
    for f, _ in FIELDS:
        cells = []
        for name in libs:
            xs = [x[f] for x in runs[name] if isinstance(x[f], (int, float))]
            st = {"median": statistics.median(xs), "min": min(xs), "max": max(xs)} if xs else None
            summary.setdefault(name, {})[f] = st
            cells.append(f"{st['median']:8.1f} [{st['min']:7.1f},{st['max']:7.1f}]" if st else f"{'n/a':>26s}")
        print(f"{f:>18s} | " + " | ".join(f"{c:>26s}" for c in cells))
    b, n = summary["base"]["value"], summary["new"]["value"]
    verdict = None
    if b and n:
        verdict = {"median_gain": n["median"] / b["median"] - 1.0, "new_min_beats_base_max": n["min"] > b["max"]}
        print(f"\nfwd+bwd median gain {100 * verdict['median_gain']:+.1f} %, new slowest > base fastest: "
              f"{verdict['new_min_beats_base_max']}")
    result = {"device": info, "seq": args.seq, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
              "libs": libs, "summary": summary, "verdict": verdict, "runs": runs, "outputs_ok": checked}
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
