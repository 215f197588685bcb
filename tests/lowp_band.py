"""Band masks for the 16-bit model and comparator of ``tests/lowp_model.py``.

The band ``("band", lo, hi)`` of ``band_oracle`` (key b visible to row a iff a + lo <= b <= a + hi, None: open side)
is what the tile kernels' band mask computes.  ``install()`` extends ``lowp_model`` in this process so that its
masks may also be bands:

* ``visible`` and ``_vis_for`` accept the band, with the model's causal mutants acting on its upper edge and the
  faults of ``BAND_MUTANTS`` on its lower edge;
* the fp64 chunk functions ``oracle_chain`` calls run through ``band_oracle``.

Every mask lowp_model already knows keeps its own code path: the replacements hand such masks to the originals.
"""
from __future__ import annotations

import torch

import band_oracle as bo
import lowp_model as lm

# One realistic fault each at the band's lower edge.  "_fwd" / "_bwd": only that kernel has the fault.
BAND_MUTANTS = (
    "band_lo_plus1_fwd",    # forward lets the key one below the band through
    "band_lo_plus1_bwd",    # backward does the same
    "band_i_end_short",     # backward: every key block skips the last Q block it should visit (i_end one block short)
)

_visible, _vis_for = lm.visible, lm._vis_for  # lowp_model's own


def visible(sq, sk, mask, device=None, shift=0, strict=False, lo_shift=0):
    """``lowp_model.visible`` extended by the band; ``lo_shift`` moves its lower edge that many keys down."""
    if mask is None or mask[0] != "band":
        return _visible(sq, sk, mask, device, shift=shift, strict=strict)
    _, lo, hi = mask
    a = torch.arange(sq, device=device).unsqueeze(1)
    b = torch.arange(sk, device=device).unsqueeze(0)
    m = torch.ones(sq, sk, dtype=torch.bool, device=device)
    if lo is not None:
        m &= b >= a + int(lo) - lo_shift
    if hi is not None:
        m &= (b < a + int(hi) + shift) if strict else (b <= a + int(hi) + shift)
    return m


def vis_for(sq, sk, mask, device, mutant, side):
    if mask is None or mask[0] != "band":
        return _vis_for(sq, sk, mask, device, mutant, side)
    shift = {"causal_plus1_" + side: 1, "causal_minus1_" + side: -1}.get(mutant, 0)
    vis = visible(sq, sk, mask, device, shift=shift, strict=mutant == "strict_swap",
                  lo_shift=1 if mutant == "band_lo_plus1_" + side else 0)
    if mutant == "band_i_end_short" and side == "bwd" and mask[1] is not None:
        # per 128-key block, the last 64-row Q block it would visit contributes nothing
        for k0 in range(0, sk, 128):
            q_last = min(k0 + 127, sk - 1) - int(mask[1])
            if q_last >= 0:
                qb = min(q_last, sq - 1) // 64 * 64
                vis[qb:qb + 64, k0:k0 + 128] = False
    return vis


class _Oracle:
    """``oracle.attention_oracle`` with chunk functions that also take the band."""

    def __init__(self, orc):
        self._orc = orc
        self.chunk_forward, self.chunk_backward = bo.chunk_forward, bo.chunk_backward

    def __getattr__(self, name):
        return getattr(self._orc, name)


def install():
    """Extend lowp_model by the band in this process (idempotent)."""
    if lm.visible is visible:
        return
    lm.visible, lm._vis_for = visible, vis_for
    lm.orc = _Oracle(lm.orc)
