"""Load the UNMODIFIED reference (MayDomine/Burst-Attention) from the git-ignored ``oracle/_ref``.

``oracle/_ref`` is written by build() through oracle/build_reference.py (a copy of the reference's pure-Python
package, where a reference checkout exists).  Nothing of it is edited or copied into the tracked tree; this file
only makes its imports resolve:

* ``bmtrain`` (absent in this image) -> a stub module, so the reference selects its torch backend
  (burst_attn/comm.py:36-37,106-114; SURVEY.md 8c);
* flash-attn's private entry points: the reference calls them with the signature of flash-attn <= 2.5
  (burst_attn/burst_utils.py:150-160,211-248); two adapters with that signature are installed on
  ``flash_attn.flash_attn_interface`` before the reference imports them (flash-attn 2.8.3 split ``window_size``,
  added ``softcap`` and returns 4 values);
* the reference package is called ``burst_attn`` like this repo's drop-in; it is loaded under the alias
  ``burst_attn_ref`` (all its intra-package imports are relative) so both can live in one process.

Users: ``bench.py`` (``cpu_baseline`` leg / ``--impl reference``: the reference's device-agnostic chunk functions on
the host cores) and ``tools/ref_on_gpu.py`` (the reference's ring on the GPUs).  Never imported by the product.
"""
import importlib.util
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")
ALIAS = "burst_attn_ref"


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "burst_attn", "__init__.py"))


def stub_bmtrain():
    if "bmtrain" in sys.modules:
        return
    bmt = types.ModuleType("bmtrain")
    bmt.init = types.SimpleNamespace(is_initialized=lambda: False)
    bmt.config = {}
    bmt.print_rank = print
    sys.modules["bmtrain"] = bmt
    d = types.ModuleType("bmtrain.distributed")
    sys.modules["bmtrain.distributed"] = d
    ops = types.ModuleType("bmtrain.distributed.ops")
    ops.ncclSend = ops.ncclRecv = None
    sys.modules["bmtrain.distributed.ops"] = ops
    nccl = types.ModuleType("bmtrain.nccl")
    for n in ("commCount", "groupEnd", "groupStart", "allReduce", "commRank"):
        setattr(nccl, n, None)
    sys.modules["bmtrain.nccl"] = nccl
    bmt.distributed, bmt.nccl = d, nccl


def adapt_flash_attn():
    """Old private signatures (what the reference calls) -> the installed flash-attn (2.8.3)."""
    import flash_attn.flash_attn_interface as fai
    if getattr(fai, "_ba_ref_adapted", False):
        return
    new_fwd, new_bwd = fai._flash_attn_forward, fai._flash_attn_backward

    def fwd_old(q, k, v, dropout_p, softmax_scale, causal, window_size=(-1, -1), alibi_slopes=None,
                return_softmax=False):
        out, lse, s_dmask, rng = new_fwd(q, k, v, dropout_p, softmax_scale, causal, window_size[0], window_size[1],
                                         0.0, alibi_slopes, return_softmax)
        return out, q, k, v, out, lse, s_dmask, rng

    def bwd_old(dout, q, k, v, out, softmax_lse, dq, dk, dv, dropout_p, softmax_scale, causal, window_size,
                alibi_slopes, deterministic, rng_state=None):
        return new_bwd(dout, q, k, v, out, softmax_lse, dq, dk, dv, dropout_p, softmax_scale, causal,
                       window_size[0], window_size[1], 0.0, alibi_slopes, deterministic, rng_state)

    fai._flash_attn_forward, fai._flash_attn_backward = fwd_old, bwd_old
    fai._ba_ref_adapted = True


def load():
    """The reference package as module ``burst_attn_ref`` (``.burst_attn_func``, ``.burst_utils`` ...)."""
    if ALIAS in sys.modules:
        return sys.modules[ALIAS]
    if not available():
        raise ImportError(f"{REF}/burst_attn not found (see the header of {__file__} for the install command)")
    stub_bmtrain()
    adapt_flash_attn()
    pkg_dir = os.path.join(REF, "burst_attn")
    spec = importlib.util.spec_from_file_location(ALIAS, os.path.join(pkg_dir, "__init__.py"),
                                                  submodule_search_locations=[pkg_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[ALIAS] = mod
    try:
        spec.loader.exec_module(mod)
    except BaseException:
        sys.modules.pop(ALIAS, None)
        raise
    return mod


# --------------------------------------------------------------------------- #
# The reference's device-agnostic chunk path on the host cores (BASELINE.md 3): the ring of W ranks simulated in
# one process with the reference's own inter_normal_attn / inter_normal_attn_backward (burst_utils.py:42-100),
# layout [B,H,S,D], schedule of OpBurstAttn.forward/backward (burst_attn_interface.py:214-248,291-396) without
# the transport (one process holds every shard).
# --------------------------------------------------------------------------- #
def cpu_ring_step(q, k, v, do, W, scale):
    """One fwd+bwd of the whole job (all W simulated ranks).  Returns (o, dq, dk, dv, seconds_fwd, seconds_bwd)."""
    import time

    import torch
    load()
    bu = sys.modules[ALIAS + ".burst_utils"]
    qs, ks, vs, dos = (t.chunk(W, dim=2) for t in (q, k, v, do))
    t0 = time.perf_counter()
    outs, lses = [], []
    for i in range(W):
        m_i = lse_i = acc_o = None
        for r in range(W):  # round r: rank i holds the K/V shard of rank (i - r) mod W
            j = (i - r) % W
            acc_o, m_i, lse_i = bu.inter_normal_attn(qs[i], ks[j], vs[j], m_i, lse_i, acc_o, scale, None)
        outs.append((acc_o * torch.exp(m_i - lse_i)).to(q.dtype))  # burst_attn_interface.py:246-250
        lses.append(lse_i)
    t1 = time.perf_counter()
    dqs = [torch.zeros_like(t) for t in qs]
    dks = [torch.zeros_like(t) for t in ks]
    dvs = [torch.zeros_like(t) for t in vs]
    deltas = [(outs[i] * dos[i]).to(torch.float32).sum(-1, keepdim=True).to(q.dtype) for i in range(W)]  # :272-278
    for j in range(W):  # K/V at home on rank j, the Q-bundle of rank i visits (reference :291-396)
        for r in range(W):
            i = (j - r) % W
            buf = torch.empty_like(qs[i])
            bu.inter_normal_attn_backward(dos[i], qs[i], ks[j], vs[j], deltas[i], lses[i].to(q.dtype), buf, dks[j],
                                          dvs[j], scale, None)
            dqs[i] += buf  # :379-382
    t2 = time.perf_counter()
    cat = lambda ts: torch.cat(list(ts), dim=2)  # noqa: E731
    return cat(outs), cat(dqs), cat(dks), cat(dvs), t1 - t0, t2 - t1
