"""The tile kernels compile for sm_90a without serialized wgmma and without register spills (no GPU needed).

ptxas serializes a kernel's whole wgmma pipeline (waits after every MMA) when the kernel makes a function call, e.g.
a printf, or when a wgmma group crosses a divergent path; it says so in an info line ("C7510" / "C7520 Potential
Performance Loss").  A spill puts local-memory traffic in the inner loop.  Both are silent slowdowns, so every
instantiation of fwd_chunk_kernel and bwd_chunk_kernel is checked here with the flags of csrc/Makefile.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "burst-attention_b200", "csrc")


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _ptxas_report(src, tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, src),
           "-o", str(tmp_path / (src + ".o"))]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return res.stderr


def _per_kernel(log, kernel):
    """{mangled name: (serialization lines, (spill stores, spill loads))} for every instantiation of `kernel`."""
    out, cur, warn = {}, None, {}
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(_Z\w+)'?", line)
        if m:
            cur = m.group(1)
        for name in re.findall(r"in the function '(_Z\w+)'", line):
            if "Performance Loss" in line or "C7510" in line:
                warn.setdefault(name, []).append(line.strip())
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and kernel in cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
    return {k: (warn.get(k, []), v) for k, v in out.items()}


@pytest.mark.parametrize("src,kernel,n_inst", [("fwd_sm90.cu", "fwd_chunk_kernel", 8),
                                               ("bwd_sm90.cu", "bwd_chunk_kernel", 4)])
def test_tile_kernels_not_serialized_and_no_spills(src, kernel, n_inst, tmp_path):
    log = _ptxas_report(src, tmp_path)
    assert "C7510" not in log and "Performance Loss" not in log, \
        "\n".join(ln for ln in log.splitlines() if "C75" in ln or "Performance Loss" in ln)
    kernels = _per_kernel(log, kernel)
    assert len(kernels) == n_inst, f"expected {n_inst} instantiations of {kernel}, found {sorted(kernels)}"
    for name, (warn, spills) in kernels.items():
        assert not warn, warn
        assert spills == (0, 0), f"{name}: {spills[0]} bytes spill stores, {spills[1]} bytes spill loads"
