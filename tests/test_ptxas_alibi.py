"""The ALiBi instantiations of the tile kernels (csrc/fwd_alibi_sm90.cu, csrc/bwd_alibi_sm90.cu) compile for sm_90a
without serialized wgmma and without register spills, as tests/test_ptxas_report.py checks for the others."""
import pytest

from test_ptxas_report import _per_kernel, _ptxas_report


@pytest.mark.parametrize("src,kernel,n_inst", [("fwd_alibi_sm90.cu", "fwd_alibi_kernel", 8),
                                               ("bwd_alibi_sm90.cu", "bwd_alibi_kernel", 8)])
def test_alibi_kernels_not_serialized_and_no_spills(src, kernel, n_inst, tmp_path):
    log = _ptxas_report(src, tmp_path)
    assert "C7510" not in log and "Performance Loss" not in log, \
        "\n".join(ln for ln in log.splitlines() if "C75" in ln or "Performance Loss" in ln)
    kernels = _per_kernel(log, kernel)
    assert len(kernels) == n_inst, f"expected {n_inst} instantiations of {kernel}, found {sorted(kernels)}"
    for name, (warn, spills) in kernels.items():
        assert not warn, warn
        assert spills == (0, 0), f"{name}: {spills[0]} bytes spill stores, {spills[1]} bytes spill loads"
