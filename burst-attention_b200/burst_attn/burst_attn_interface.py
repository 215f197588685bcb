"""Public API and ring drivers: ``burst_attn_func`` / ``burst_attn_func_striped``
with the reference's positional signature (burst_attn_interface.py:109-158), as
``torch.autograd.Function``s ``OpBurstAttn`` / ``OpBurstAttnStrip`` (:161-613).

What is the same as the reference: names, argument order and defaults, shard
layouts (contiguous / zigzag halves / striped, test/test_burst.py:44-58), the
ring schedules (forward: K/V rotate, :214-242; backward: the Q-bundle
(delta, dO, Q, lse) rotates and the partial dQ rides one hop behind it,
:291-396), output dtype, the assertion that causal needs flash == "cuda".  The hierarchical ("double")
ring (reference comm.py:187-254) runs through the same two drivers (``_ring_forward`` / ``_bwd_rounds``):
the flat ring is its special case of one node.

What is H100-native instead (DESIGN.md): every round is ONE kernel launch of the
C-ABI library (carried (O, lse) state and fp32 dQ/dK/dV accumulation fused into
the tile kernels; half-sequence and shifted cases are pointer/length views or a
causal offset, never ``.contiguous()`` copies); user tensors are never used as
receive buffers; the ring hop is grouped NCCL send/recv on a side stream posted
before the round's kernel and awaited after it.
"""
from __future__ import annotations

import math
import os
from typing import List

import torch

from .chunk_ops import get_ops
from .comm import Ring, get_rank, get_world_size

__all__ = ["burst_attn_func", "burst_attn_func_striped", "OpBurstAttn", "OpBurstAttnStrip",
           "get_partition_id", "split2_gethalf"]


class _Range:
    """NVTX range per ring round (BA_NVTX=1): `ncu --nvtx --nvtx-include "bwd_round_3/"` or a timeline tool then
    sees the post / kernel / wait of one round as a unit (SURVEY.md 5.1).  A no-op otherwise."""
    on = os.environ.get("BA_NVTX", "0") == "1"

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if _Range.on:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if _Range.on:
            torch.cuda.nvtx.range_pop()
        return False


def get_partition_id(double_group, r):
    """Reference :20-37.  Single ring (``double_group[0] is None``): the OFFSET ``r - 1`` of the held shard
    behind this rank.  Double ring: the RANK ID of the held shard, ``W = L*M``, rank ``= inter*L + intra``:
    node ``(inter - (r-1)//L) mod M``, slot ``(intra - (r-1)%L) mod L`` (SURVEY.md Appendix C)."""
    if double_group[0] is None:
        return r - 1
    L, M = get_world_size(double_group[0]), get_world_size(double_group[1])
    b, a = get_rank(double_group[0]), get_rank(double_group[1])
    return ((a - (r - 1) // L) % M) * L + (b - (r - 1) % L) % L


# Hierarchical ring over NCCL: on when the caller passes double_group (BA_DOUBLE_RING=0 forces the flat ring over
# process_group).  `RING_CHECK_DOUBLE=2,4 torchrun tests/ring_check.py` checks it for intra-node rings of 2 and of 4.
_DOUBLE_RING_DEFAULT = "1"


class _Topology:
    """Ring topology of one call: flat (one ring over ``process_group``) or hierarchical
    (``double_group = [intra, inter]``, each optionally a ``(group, dq_group)`` pair, reference :188-194)."""

    def __init__(self, process_group, double_group):
        self.group = process_group
        self.W, self.rank = get_world_size(process_group), get_rank(process_group)
        intra, inter = double_group[0], double_group[1]
        self.intra_dq = self.inter_dq = None
        if isinstance(intra, (tuple, list)):
            intra, self.intra_dq = intra
        if isinstance(inter, (tuple, list)):
            inter, self.inter_dq = inter
        self.intra, self.inter = intra, inter
        self.L, self.M = self.W, 1
        self.hier = False
        if intra is not None and inter is not None and os.environ.get("BA_DOUBLE_RING", _DOUBLE_RING_DEFAULT) != "0":
            L, M = get_world_size(intra), get_world_size(inter)
            if 1 < L < self.W:  # reference comm.py:215-219: a ring that is all-intra (or all-inter) is flat
                assert L * M == self.W, f"double ring: intra size {L} x inter size {M} != world {self.W}"
                self.a, self.b = get_rank(inter), get_rank(intra)
                assert self.a * L + self.b == self.rank, "double ring expects rank = inter_rank * intra_size + intra_rank"
                self.L, self.M, self.hier = L, M, True

    def source(self, r):
        """Rank whose shard (K/V forward, Q-bundle backward) is held in round r (1-based)."""
        if not self.hier:
            return (self.rank - (r - 1)) % self.W
        return get_partition_id([self.intra, self.inter], r)

    def rings(self):
        """(ring, inter, inter_dq): the ring the blocks hop round inside a cycle, and on the hierarchical ring the
        inter-node rings of the block prefetch and of the dQ node sums (None on the flat ring)."""
        if not self.hier:
            return Ring(self.group, tag="ring"), None, None
        # the copy-engine transport serves the flat ring only: its receive buffers are tied to one ring's arena
        return (Ring(self.intra, tag="ring", transport="nccl"), Ring(self.inter, tag="inter", transport="nccl"),
                Ring(self.inter_dq if self.inter_dq is not None else self.inter, tag="inter_dq", transport="nccl"))


def split2_gethalf(inp, first_dim, half_idx=0):
    """Half-sequence VIEW (reference :96-106); never copied here."""
    dim = 1 if first_dim else 2
    n = inp.shape[dim] // 2
    return inp.narrow(dim, 0, n) if half_idx == 0 else inp.narrow(dim, n, inp.shape[dim] - n)


def _half(t, dim, idx):
    n = t.shape[dim] // 2
    return t.narrow(dim, 0, n) if idx == 0 else t.narrow(dim, n, t.shape[dim] - n)


def _nbytes(t) -> int:
    return t.numel() * t.element_size()


def _l2_block() -> int:
    """Rows/keys per sub-launch.  One (batch, head) slice of 32768 keys is 16 MiB of K+V (or 32 MiB of
    Q, dO and fp32 dQ in the backward), so the streamed operands of a launch can stay resident in H100's
    50 MB L2 while all CTAs of a head sweep them.  The multi-GPU rounds at S_local <= 49152 are unaffected.  BA_L2_BLOCK overrides (tests use tiny blocks)."""
    return int(os.environ.get("BA_L2_BLOCK", "32768"))


def _bias_kw(bias, c0=None, n=None):
    """Keyword for the chunk operators: the key-bias view of keys [c0, c0+n) (nothing when there is no bias, so
    test operators without a bias parameter keep working)."""
    if bias is None:
        return {}
    return {"bias": bias if c0 is None else bias.narrow(2, c0, n)}


def _fwd_round(ops, q, k, v, o_acc, lse, out, scale, causal, off, first, last, seq_dim, bias=None):
    """One forward ring round, split over K/V blocks that fit L2 (each block is one kernel launch with
    the carried state; the state pass costs 2 x 512 B per row and head, the block > 8 MB of math)."""
    blk = _l2_block()
    if k.shape[seq_dim] <= blk + blk // 2:
        ops.fwd_chunk(q, k, v, o_acc, lse, out, scale, causal, off, first, last, seq_dim, **_bias_kw(bias))
        return
    _fwd_blocks(ops, q, k, v, o_acc, lse, out, scale, causal, off, first, last, seq_dim, blk, bias)


def _fwd_blocks(ops, q, k, v, o_acc, lse, out, scale, causal, off, first, last, seq_dim, blk, bias=None,
                before=None):
    """A forward round as one launch per block of ``blk`` keys; ``before(c)``, if given, runs first in the step
    of block c (host_stream.py waits there for the block's upload)."""
    Sq, Sk = q.shape[seq_dim], k.shape[seq_dim]
    n = (Sk + blk - 1) // blk
    for c in range(n):
        c0 = c * blk
        kc, vc = k.narrow(seq_dim, c0, min(blk, Sk - c0)), v.narrow(seq_dim, c0, min(blk, Sk - c0))
        if before is not None:
            before(c)
        if not causal:
            ops.fwd_chunk(q, kc, vc, o_acc, lse, out, scale, False, 0, first and c == 0, last and c == n - 1, seq_dim,
                          **_bias_kw(bias, c0, min(blk, Sk - c0)))
            continue
        # causal: rows before r_start see none of this block's keys (key c0+b visible to row a iff
        # c0 + b <= a + off); keep r_start on a tile-pair boundary
        r_start = max(0, (c0 - off) // 256 * 256)
        if r_start >= Sq:
            break
        ops.fwd_chunk(q.narrow(seq_dim, r_start, Sq - r_start), kc, vc,
                      o_acc.narrow(seq_dim, r_start, Sq - r_start), lse.narrow(2, r_start, Sq - r_start), None,
                      scale, True, r_start + off - c0, first and c == 0, False, seq_dim,
                      **_bias_kw(bias, c0, min(blk, Sk - c0)))
    if causal and last:
        ops.cast(o_acc, out, seq_dim)


def _fwd_round_needs_state(k, seq_dim) -> bool:
    blk = _l2_block()
    return k.shape[seq_dim] > blk + blk // 2


def _bwd_round(ops, g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, causal, off, seq_dim, deterministic,
               bias=None):
    """One backward ring round, split over blocks of Q-bundle rows that fit L2."""
    blk = _l2_block()
    Sq = q.shape[seq_dim]
    if Sq <= blk + blk // 2:
        ops.bwd_chunk(g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, causal, off, seq_dim, deterministic,
                      **_bias_kw(bias))
        return
    for r0 in range(0, Sq, blk):
        _bwd_rows(ops, g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, causal, off, seq_dim, deterministic,
                  r0, min(blk, Sq - r0), bias)


def _bwd_rows(ops, g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, causal, off, seq_dim, deterministic,
              r0, n, bias=None):
    """Rows [r0, r0+n) of a backward round as one launch over the keys they see (none: no launch)."""
    kk, vv, dk, dv, o2, bkw = k, v, dk_acc, dv_acc, off, _bias_kw(bias)
    if causal:
        kmax = min(k.shape[seq_dim], r0 + n + off)  # keys visible to the last row of this block
        if kmax <= 0:
            return
        kk, vv, bkw = k.narrow(seq_dim, 0, kmax), v.narrow(seq_dim, 0, kmax), _bias_kw(bias, 0, kmax)
        dk, dv = dk_acc.narrow(seq_dim, 0, kmax), dv_acc.narrow(seq_dim, 0, kmax)
        o2 = off + r0
    ops.bwd_chunk(g.narrow(seq_dim, r0, n), q.narrow(seq_dim, r0, n), kk, vv, delta.narrow(2, r0, n),
                  lse.narrow(2, r0, n), dq_part.narrow(seq_dim, r0, n), dk, dv, scale, causal, o2, seq_dim,
                  deterministic, **bkw)


# --------------------------------------------------------------------------- #
# sliding-window (local) attention: band masks per round
# --------------------------------------------------------------------------- #
def _check_window(window_size, causal):
    """flash-attn's ``window_size=(left, right)`` (-1: that side unlimited; ``causal`` forces right = 0) ->
    ``(left, right)`` with None for an unlimited side, or None when nothing is windowed: such a call runs exactly as
    one without the argument."""
    if window_size is None:
        return None
    try:
        left, right = (int(x) for x in window_size)
    except (TypeError, ValueError):
        raise ValueError(f"window_size must be a pair (left, right) of ints, got {window_size!r}") from None
    for name, x in (("left", left), ("right", right)):
        if x < -1:
            raise ValueError(f"window_size: {name} = {x}; it must be -1 (unlimited) or >= 0")
    left = None if left == -1 else left
    right = 0 if causal else (None if right == -1 else right)
    if left is None and (right is None or causal):
        return None
    return left, right


def _band(qn, kn, lo, hi):
    """The band of a view of ``qn`` rows and ``kn`` keys -- key c visible to row a iff a + lo <= c <= a + hi (None:
    that side open) -- with the sides that mask nothing opened, or None when no row sees any key (no launch)."""
    if hi is not None and (qn - 1 + hi < 0 or (lo is not None and lo > hi)):
        return None
    if lo is not None and lo >= kn:
        return None
    if hi is not None and hi >= kn - 1:
        hi = None
    if lo is not None and lo <= 1 - qn:
        lo = None
    return lo, hi


def _round_pieces(layout, W, iq, jk, S, window):
    """The pieces of the round that attends the Q shard of rank ``iq`` to the K/V shard of rank ``jk`` (``S`` rows
    each): ``[(q0, qn, k0, kn, lo, hi)]``, rows and keys local to the shards, the band relative to the two views;
    pieces whose band misses its view are left out.  ``window`` = (left, right) counts positions in the full
    sequence: contiguous shards start at rank * S, zigzag shards are the halves rank and 2W-1-rank (one piece per
    pair of halves), and striped token a of rank r sits at a W + r, so a + ceil((iq-jk-left)/W) <= c <=
    a + floor((iq-jk+right)/W)."""
    left, right = window
    if layout == "striped":
        cand = [(0, S, 0, S, None if left is None else -((jk - iq + left) // W),
                 None if right is None else (iq - jk + right) // W)]
    else:
        if layout == "contiguous":
            qs, ks = [(0, S, iq * S)], [(0, S, jk * S)]
        else:
            assert S % 2 == 0, "zigzag causal sharding needs an even local sequence length"
            h = S // 2
            qs = [(0, h, iq * h), (h, h, (2 * W - 1 - iq) * h)]
            ks = [(0, h, jk * h), (h, h, (2 * W - 1 - jk) * h)]
        cand = [(qa, qn, ka, kn, None if left is None else qg - kg - left, None if right is None else qg - kg + right)
                for qa, qn, qg in qs for ka, kn, kg in ks]
    out = []
    for qa, qn, ka, kn, lo, hi in cand:
        b = _band(qn, kn, lo, hi)
        if b is not None:
            out.append((qa, qn, ka, kn) + b)
    return out


def _fwd_band_launches(pieces):
    """Forward launches ``[(q0, qn, k0, kn, lo, hi)]`` of a round's pieces: a piece longer than the L2 block is split
    over blocks of keys as in ``_fwd_blocks``, each launch taking only the rows that see its block."""
    blk = _l2_block()
    out = []
    for qa, qn, ka, kn, lo, hi in pieces:
        if kn <= blk + blk // 2:
            out.append((qa, qn, ka, kn, lo, hi))
            continue
        for c0 in range(0, kn, blk):
            cn = min(blk, kn - c0)
            r0 = 0 if hi is None else max(0, c0 - hi)
            r1 = qn if lo is None else min(qn, c0 + cn - lo)
            b = _band(r1 - r0, cn, None if lo is None else lo + r0 - c0, None if hi is None else hi + r0 - c0) \
                if r0 < r1 else None
            if b is not None:
                out.append((qa + r0, r1 - r0, ka + c0, cn) + b)
    return out


def _bwd_band_launches(pieces):
    """Backward launches of a round's pieces: a piece with more rows than the L2 block is split over blocks of rows
    as in ``_bwd_rows``, each launch taking only the keys its rows see."""
    blk = _l2_block()
    out = []
    for qa, qn, ka, kn, lo, hi in pieces:
        if qn <= blk + blk // 2:
            out.append((qa, qn, ka, kn, lo, hi))
            continue
        for r0 in range(0, qn, blk):
            rn = min(blk, qn - r0)
            c0 = 0 if lo is None else max(0, r0 + lo)
            c1 = kn if hi is None else min(kn, r0 + rn + hi)
            b = _band(rn, c1 - c0, None if lo is None else lo + r0 - c0, None if hi is None else hi + r0 - c0) \
                if c0 < c1 else None
            if b is not None:
                out.append((qa + r0, rn, ka + c0, c1 - c0) + b)
    return out


def _lower_kw(lo):
    """Keyword for the chunk operators: the band's lower edge (nothing without one)."""
    return {} if lo is None else {"lower": lo}


# --------------------------------------------------------------------------- #
# ALiBi: -slope |pos_q - pos_k| over positions of the full sequence
# --------------------------------------------------------------------------- #
def _check_alibi(alibi_slopes, q, heads_dim):
    """flash-attn's ``alibi_slopes`` (fp32, ``(nheads,)`` or ``(batch, nheads)``, on q's device) -> an fp32 [B, H]
    view (stride 0 over the batch for one row), or None."""
    if alibi_slopes is None:
        return None
    B, H = q.shape[0], q.shape[heads_dim]
    if not isinstance(alibi_slopes, torch.Tensor):
        raise TypeError(f"alibi_slopes must be a torch.Tensor, got {type(alibi_slopes).__name__}")
    if alibi_slopes.dtype != torch.float32:
        raise TypeError(f"alibi_slopes must be float32, got {alibi_slopes.dtype}")
    if alibi_slopes.device != q.device:
        raise ValueError(f"alibi_slopes is on {alibi_slopes.device}, q on {q.device}")
    if tuple(alibi_slopes.shape) not in ((H,), (B, H)):
        raise ValueError(f"alibi_slopes must have shape ({H},) or ({B}, {H}), got {tuple(alibi_slopes.shape)}")
    if not bool(torch.isfinite(alibi_slopes).all()):
        raise ValueError("alibi_slopes must be finite")
    s = alibi_slopes.detach().contiguous()
    return s.unsqueeze(0).expand(B, H) if s.dim() == 1 else s


def _positions(layout, W, rank, S):
    """Full-sequence position of local token x of ``rank``'s shard (``S`` tokens), as a function, and the distance
    between neighbouring tokens.  ``layout`` "local" is one device's view; its rank is the offset of row 0."""
    if layout == "striped":
        return (lambda x: x * W + rank), W
    if layout == "zigzag":
        h = S // 2
        return (lambda x: (rank * h + x) if x < h else ((2 * W - 1 - rank) * h + x - h)), 1
    if layout == "local":
        return (lambda x: x + rank), 1
    return (lambda x: rank * S + x), 1


def _alibi_kw(alibi, q0, k0):
    """Keyword for the chunk operators: the ALiBi of the launch whose rows start at local row q0 and keys at local
    key k0.  alibi: (slopes, pos_q, pos_k, pstride) with the position functions of ``_positions`` (or None)."""
    if alibi is None:
        return {}
    slopes, pos_q, pos_k, pstride = alibi
    return {"alibi": (slopes, pos_q(q0) - pos_k(k0), pstride)}


def _alibi_window(window, causal, alibi):
    """A call with ALiBi runs the band launches (they know where their rows and keys sit), with the unwindowed band
    when there is no window."""
    if alibi is None or window is not None:
        return window
    return (None, 0 if causal else None)


def _ring_alibi(slopes, layout, W, iq, jk, S):
    """The ALiBi of the round that attends the Q shard of rank iq to the K/V shard of rank jk (or None)."""
    if slopes is None:
        return None
    pos_q, pstride = _positions(layout, W, iq, S)
    pos_k, _ = _positions(layout, W, jk, S)
    return slopes, pos_q, pos_k, pstride


class _BandForward:
    """The launches of a windowed forward, known up front for every round, and their first / last duties.  Skipped
    launches must not drop either: the state is started by the first launch only if it covers every row (otherwise
    it starts as O = 0, lse = -inf in memory), and the output is written by the last launch only if it covers every
    row (otherwise it is cast from the fp32 state at the end)."""

    def __init__(self, rounds, q, lse, S):
        flat = [x for launches in rounds for x in launches]
        full = lambda x: x[0] == 0 and x[1] == S  # noqa: E731
        self.first = bool(flat) and full(flat[0])
        self.last = bool(flat) and full(flat[-1])
        self.n, self.done = len(flat), 0
        self.o_acc = None
        if not (self.n == 1 and self.first and self.last):
            self.o_acc = torch.empty(q.shape, dtype=torch.float32, device=q.device)
        if not self.first:
            self.o_acc.zero_()
            lse.fill_(float("-inf"))

    def run(self, ops, launches, q, k, v, lse, out, scale, seq_dim, bias=None, alibi=None):
        for q0, qn, k0, kn, lo, hi in launches:
            first = self.first and self.done == 0
            last = self.last and self.done == self.n - 1
            rows = lambda t: t.narrow(seq_dim, q0, qn)  # noqa: E731
            ops.fwd_chunk(rows(q), k.narrow(seq_dim, k0, kn), v.narrow(seq_dim, k0, kn),
                          None if self.o_acc is None else rows(self.o_acc), lse.narrow(2, q0, qn),
                          rows(out) if last else None, scale, hi is not None, 0 if hi is None else hi, first, last,
                          seq_dim, **_bias_kw(bias, k0, kn), **_lower_kw(lo), **_alibi_kw(alibi, q0, k0))
            self.done += 1

    def finish(self, ops, out, seq_dim):
        if not self.last:
            ops.cast(self.o_acc, out, seq_dim)


def _bwd_band_run(ops, launches, g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, seq_dim, deterministic,
                  bias=None, alibi=None):
    for q0, qn, k0, kn, lo, hi in launches:
        rows = lambda t: t.narrow(seq_dim, q0, qn)  # noqa: E731
        keys = lambda t: t.narrow(seq_dim, k0, kn)  # noqa: E731
        ops.bwd_chunk(rows(g), rows(q), keys(k), keys(v), delta.narrow(2, q0, qn), lse.narrow(2, q0, qn),
                      rows(dq_part), keys(dk_acc), keys(dv_acc), scale, hi is not None, 0 if hi is None else hi, seq_dim,
                      deterministic, **_bias_kw(bias, k0, kn), **_lower_kw(lo), **_alibi_kw(alibi, q0, k0))


def _check_inputs(q, k, v, seq_dim):
    assert q.dim() == 4 and k.shape == v.shape and q.shape[0] == k.shape[0] and q.shape[3] == k.shape[3], \
        "q, k, v must be 4-D with matching batch and head_dim"
    hq, hkv = q.shape[3 - seq_dim], k.shape[3 - seq_dim]
    assert hkv > 0 and hq % hkv == 0, \
        f"the number of q heads ({hq}) must be a multiple of the number of k/v heads ({hkv})"
    assert q.dtype == k.dtype == v.dtype, "q, k, v must share a dtype"


def _fwd_dispatch(ops, mode, r, W, i, j, q, cur_k, cur_v, o_acc, lse, out, scale, seq_dim):
    """The kernel work of forward round r on rank i holding the K/V shard of rank j (SURVEY.md App. B)."""
    first, last = r == 1, r == W
    if mode == "none":
        _fwd_round(ops, q, cur_k, cur_v, o_acc, lse, out, scale, False, 0, first, last, seq_dim)
    elif mode == "zigzag":
        if r == 1:  # own shard: plain causal (:221-224)
            _fwd_round(ops, q, cur_k, cur_v, o_acc, lse, out, scale, True, 0, first, last, seq_dim)
        elif j < i:  # split_kv: all Q x first half of K/V (:225-231)
            _fwd_round(ops, q, _half(cur_k, seq_dim, 0), _half(cur_v, seq_dim, 0), o_acc, lse, out, scale,
                       False, 0, False, last, seq_dim)
        else:  # second half of Q x all K/V, merged into the second half of the state (:232-235)
            _fwd_round(ops, _half(q, seq_dim, 1), cur_k, cur_v, _half(o_acc, seq_dim, 1), _half(lse, 2, 1),
                       _half(out, seq_dim, 1), scale, False, 0, False, last, seq_dim)
            if last:  # rows the last round did not visit: hand their finished state over
                ops.cast(_half(o_acc, seq_dim, 0), _half(out, seq_dim, 0), seq_dim)
    elif mode == "striped":
        # source rank ahead of us -> strictly-lower-triangular (causal_shift, :454,:463-475)
        _fwd_round(ops, q, cur_k, cur_v, o_acc, lse, out, scale, True, -1 if j > i else 0, first, last, seq_dim)
    else:
        raise ValueError(mode)


# --------------------------------------------------------------------------- #
# forward ring (reference OpBurstAttn.forward :171-253, OpBurstAttnStrip.forward :411-493)
# --------------------------------------------------------------------------- #
def _ring_forward(q, k, v, scale, seq_dim, mode, topo, window=None, layout=None, alibi=None):
    """mode: "none" (non-causal) | "zigzag" | "striped".  Returns (out, lse[B,H,S] fp32).  With a ``window``
    (``_check_window``) the rounds run the band launches of ``_round_pieces`` for the shard ``layout`` instead.

    Rounds run in M cycles of L steps (the flat ring is one cycle, L = W).  Within a cycle K/V hop round the
    intra-node ring; on the hierarchical ring (reference comm.py:187-254, SURVEY.md Appendix C) the block a
    cycle starts with is at the same time forwarded to the next node over the inter-node ring, where it starts
    the following cycle -- a prefetch with L rounds of kernel time to hide behind.  Unlike the reference no
    send-side copy is made: the cycle's starting block is never a receive target while it is in flight (two
    inter-node buffers alternate).

    ``alibi`` (fp32 slopes [B, H] from ``_check_alibi``) runs the band launches too, with the unwindowed band when
    there is no window, so that every launch knows where its rows and keys sit in the full sequence."""
    ops = get_ops()
    window = _alibi_window(window, mode != "none", alibi)
    ring, inter, _ = topo.rings()
    L, M, W, i = topo.L, topo.M, topo.W, topo.rank
    B, S, H = q.shape[0], q.shape[seq_dim], q.shape[3 - seq_dim]
    if mode == "zigzag":
        assert S % 2 == 0, "zigzag causal sharding needs an even local sequence length"
    out = torch.empty_like(q)
    lse = torch.empty((B, H, S), dtype=torch.float32, device=q.device)
    band = None
    if window is not None:
        band = _BandForward([_fwd_band_launches(_round_pieces(layout, W, i, topo.source(r), S, window))
                             for r in range(1, W + 1)], q, lse, S)
        o_acc = None
    else:
        need_state = W > 1 or _fwd_round_needs_state(k, seq_dim)
        o_acc = torch.empty(q.shape, dtype=torch.float32, device=q.device) if need_state else None
    if W > 1:
        k, v = k.contiguous(), v.contiguous()
    ring.begin(q, [_nbytes(k), _nbytes(v)] * min(2, L - 1))
    recv = [[ring.empty_like(k), ring.empty_like(v)] for _ in range(min(2, L - 1))]
    xbuf = [[torch.empty_like(k), torch.empty_like(v)] for _ in range(min(2, M - 1))]
    cur = [k, v]
    for r in range(1, W + 1):
        c, t = divmod(r - 1, L)
        j = topo.source(r)  # source rank of the held K/V (App. B)
        with _Range(f"fwd_round_{r}"):
            if t == 0 and c != M - 1:  # next cycle's starting block, from the previous node
                inter.post(cur, xbuf[c % len(xbuf)])
            if t != L - 1:
                nxt = recv[(r - 1) % len(recv)]
                ring.post(cur, nxt)
            if band is None:
                _fwd_dispatch(ops, mode, r, W, i, j, q, cur[0], cur[1], o_acc, lse, out, scale, seq_dim)
            else:  # a round whose shard lies outside every row's window launches nothing
                band.run(ops, _fwd_band_launches(_round_pieces(layout, W, i, j, S, window)), q, cur[0], cur[1], lse,
                         out, scale, seq_dim, alibi=_ring_alibi(alibi, layout, W, i, j, S))
            if t != L - 1:
                ring.wait()
                cur = nxt
            elif c != M - 1:
                inter.wait()
                cur = xbuf[c % len(xbuf)]
    if band is not None:
        band.finish(ops, out, seq_dim)
    return out, lse


# --------------------------------------------------------------------------- #
# backward ring (reference OpBurstAttn.backward :256-398, OpBurstAttnStrip.backward :496-613)
# --------------------------------------------------------------------------- #
def _bwd_dispatch(ops, mode, r, i, j, bundle, dq_part, k, v, dk_acc, dv_acc, scale, seq_dim, deterministic):
    """The kernel work of backward round r: K/V at home on rank i, Q-bundle of rank j (SURVEY.md App. B)."""
    dlt, g, qq, ls = bundle
    if mode == "none":
        _bwd_round(ops, g, qq, k, v, dlt, ls, dq_part, dk_acc, dv_acc, scale, False, 0, seq_dim, deterministic)
    elif mode == "zigzag":
        if r == 1:
            _bwd_round(ops, g, qq, k, v, dlt, ls, dq_part, dk_acc, dv_acc, scale, True, 0, seq_dim, deterministic)
        elif j < i:  # split_q: second half of the bundle x all K/V (:322-345,:383-386)
            _bwd_round(ops, _half(g, seq_dim, 1), _half(qq, seq_dim, 1), k, v, _half(dlt, 2, 1), _half(ls, 2, 1),
                       _half(dq_part, seq_dim, 1), dk_acc, dv_acc, scale, False, 0, seq_dim, deterministic)
        else:  # whole bundle x first half of K/V (:347-367,:387-390)
            _bwd_round(ops, g, qq, _half(k, seq_dim, 0), _half(v, seq_dim, 0), dlt, ls, dq_part,
                       _half(dk_acc, seq_dim, 0), _half(dv_acc, seq_dim, 0), scale, False, 0, seq_dim,
                       deterministic)
    elif mode == "striped":
        # K/V home on i, bundle from j: strict iff j < i (causal_shift, :529)
        _bwd_round(ops, g, qq, k, v, dlt, ls, dq_part, dk_acc, dv_acc, scale, True, -1 if j < i else 0, seq_dim,
                   deterministic)
    else:
        raise ValueError(mode)


def _ring_backward(d_o, q, k, v, out, lse, scale, seq_dim, mode, topo, deterministic, window=None, layout=None,
                   alibi=None):
    ops = get_ops()
    window = _alibi_window(window, mode != "none", alibi)
    W, i = topo.W, topo.rank
    dev = q.device
    q, k, v, d_o, out = (t.contiguous() for t in (q, k, v, d_o, out))
    B, S, H = q.shape[0], q.shape[seq_dim], q.shape[3 - seq_dim]

    # delta always travels instead of O (the reference's optimize_bwd_comm, :271-278):
    # 4 B instead of 2*D B per row and head, and the tile kernel never needs O.
    delta = torch.empty((B, H, S), dtype=torch.float32, device=dev)
    ops.delta(out, d_o, delta, seq_dim)

    f32 = dict(dtype=torch.float32, device=dev)
    dk_acc = torch.zeros(k.shape, **f32)
    dv_acc = torch.zeros(v.shape, **f32)

    def round_kernel(r, j, bundle, dq_part):
        if window is None:
            _bwd_dispatch(ops, mode, r, i, j, bundle, dq_part, k, v, dk_acc, dv_acc, scale, seq_dim, deterministic)
            return
        dlt, g, qq, ls = bundle  # the bundle of rank j against the K/V at home: rows of j, keys of i
        _bwd_band_run(ops, _bwd_band_launches(_round_pieces(layout, W, j, i, S, window)), g, qq, k, v, dlt, ls,
                      dq_part, dk_acc, dv_acc, scale, seq_dim, deterministic,
                      alibi=_ring_alibi(alibi, layout, W, j, i, S))

    bundle = [delta, d_o, q, lse.contiguous()]
    if W == 1:
        dq_final = torch.zeros(q.shape, **f32)
        round_kernel(1, i, bundle, dq_final)
    else:
        dq_final = _bwd_rounds(ops, topo, round_kernel, bundle, q, seq_dim)

    dq = torch.empty_like(q)
    dk = torch.empty_like(k)
    dv = torch.empty_like(v)
    ops.cast(dq_final, dq, seq_dim)
    ops.cast(dk_acc, dk, seq_dim)
    ops.cast(dv_acc, dv, seq_dim)
    return dq, dk, dv


def _bwd_rounds(ops, topo, round_kernel, bundle, q, seq_dim):
    """Backward rounds over the ring (W > 1, M cycles of L steps as in the forward); returns the fp32 dQ of
    this rank's own rows.

    The Q-bundle travels exactly like K/V in the forward (hops inside a cycle; on the hierarchical ring the
    cycle's starting bundle is prefetched to the next node).  Its dQ comes home in two levels (the
    reference's ``double_ring_send_recv_q``, comm.py:187-213, restated):
      * inside a cycle the partial rides one hop behind its bundle (:300-302) and picks up each rank's
        contribution; one more hop after the cycle's last step closes the ring, so the NODE sum for a bundle
        lands on the rank that started it in this node -- on the flat ring that is the hop home (:393-396);
      * on the hierarchical ring node sums chain along the inter-node ring: at the start of cycle c the node
        sum of the bundle started in cycle c-1 is added to the running sum received from the previous node
        and sent on -- L rounds of kernel time to hide behind.  After the last cycle the same step is the hop
        home.
    """
    L, M, W = topo.L, topo.M, topo.W
    ring, inter, inter_q = topo.rings()
    dev = q.device
    # every buffer that is ever the destination of a hop on `ring` comes from it (the copy-engine transport
    # keeps them in its IPC-mapped arena): two bundle sets and the three rotating fp32 dQ buffers, all the
    # flat ring ever takes; only the hierarchical ring's node-sum chain takes more
    ring.begin(q, [_nbytes(t) for t in bundle] * min(2, L - 1) + [4 * q.numel()] * 3)
    recv = [[ring.empty_like(t) for t in bundle] for _ in range(min(2, L - 1))]
    xbuf = [[torch.empty_like(t) for t in bundle] for _ in range(min(2, M - 1))]
    part = ring.empty(q.shape, torch.float32, dev)  # this round's dQ partial (the kernel reduce-adds into it)
    part.zero_()
    free = [ring.empty(q.shape, torch.float32, dev), ring.empty(q.shape, torch.float32, dev)]

    def take():
        return free.pop() if free else ring.empty(q.shape, torch.float32, dev)

    hold = None      # dQ accumulated in this node for the bundle held in the previous round
    running = None   # inter-node running sum in flight to the next node (kept alive until awaited)
    inter_in = None  # running sum arriving from the previous node

    def chain(node_sum):
        """node_sum (+ the sum received from the previous node) -> next node; returns the receive buffer."""
        nonlocal running, inter_in
        if inter_in is not None:
            inter_q.wait()
            ops.accumulate(inter_in, node_sum, seq_dim)
            free.extend([inter_in, running])
        running, inter_in = node_sum, take()
        inter_q.post([running], [inter_in])

    for r in range(1, W + 1):
        c, t = divmod(r - 1, L)
        j = topo.source(r)
        srcs: List[torch.Tensor] = []
        dsts: List[torch.Tensor] = []
        if t != L - 1:  # bundle hop (:295-299)
            nxt = recv[(r - 1) % len(recv)]
            srcs += bundle
            dsts += nxt
        if r != 1:  # dQ hop: behind its bundle (t > 0), or closing the previous cycle's ring (t == 0)
            inbound = take()
            srcs.append(hold)
            dsts.append(inbound)
        with _Range(f"bwd_round_{r}"):
            if srcs:
                ring.post(srcs, dsts)
            if t == 0 and c != M - 1:  # next cycle's starting bundle, from the previous node
                inter.post(bundle, xbuf[c % len(xbuf)])
            round_kernel(r, j, bundle, part)
            if srcs:
                ring.wait()
        if t == 0:
            if r != 1:
                free.append(hold)
                chain(inbound)  # inbound = node sum of the bundle this rank started one cycle ago
            hold, part = part, take()
            part.zero_()
        else:
            ops.accumulate(part, inbound, seq_dim)  # dq += buf (:379-390), in fp32
            free.append(hold)
            hold = inbound
            if r != W:
                part.zero_()
        if t != L - 1:
            bundle = nxt
        elif c != M - 1:
            inter.wait()
            bundle = xbuf[c % len(xbuf)]
    # close the last cycle's ring; on the hierarchical ring the last inter-node hop is then the hop home
    home = take()
    ring.post([hold], [home])
    ring.wait()
    if M > 1:
        chain(home)
        inter_q.wait()
        home = inter_in
    return home


# --------------------------------------------------------------------------- #
def _prepare(ctx, q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic, process_group,
             double_group, window_size=(-1, -1), alibi_slopes=None):
    assert not causal or flash == "cuda", "Causal attention only supported for Flash v2"
    ctx.window = _check_window(window_size, causal)
    ctx.alibi = _check_alibi(alibi_slopes, q, 2 if flash in ["cuda", "triton"] else 1)
    ctx.softmax_scale = 1 / math.sqrt(q.shape[-1]) if softmax_scale is None else softmax_scale
    ctx.flash = None if flash not in ["cuda", "triton"] else flash
    ctx.seq_dim = 1 if ctx.flash else 2
    ctx.causal = causal
    ctx.optimize_bwd_comm = optimize_bwd_comm  # delta always travels; kept for API parity
    ctx.deterministic = deterministic
    ctx.process_group = process_group
    ctx.double_group = double_group
    ctx.topo = _Topology(process_group, double_group)
    _check_inputs(q, k, v, ctx.seq_dim)


def _pad_head_dim(ops, tensors):
    """The sm_90a tile kernels exist for head_dim 64 and 128 (``ops.tile_head_dims``; the reference's
    CPU-runnable configuration C1 has 64, its benchmarks 128).  Any other head_dim <= 128 is run exactly by
    zero-padding the last axis once per call up to the next tile width: padded Q/K columns add 0 to every score,
    padded V columns produce output columns that are exactly 0 and are sliced off, and the same holds for
    dO -> dQ/dK/dV."""
    tiles = getattr(ops, "tile_head_dims", None)
    D = tensors[0].shape[-1]
    if tiles is None or D in tiles:
        return tensors, D
    bigger = [t for t in tiles if t > D]
    assert bigger, f"head_dim {D} > {max(tiles)} is not supported"
    return [torch.nn.functional.pad(t, (0, min(bigger) - D)) for t in tensors], D


def _unpad(t, D):
    return t if t.shape[-1] == D else t[..., :D].contiguous()


def _op_forward(ctx, q, k, v, mode, layout):
    """mode: the schedule of the call without a window; layout: its shards ("contiguous" | "zigzag" | "striped"),
    which a window needs even where the mask-free schedule does not."""
    ctx.host = False
    if q.device.type == "cpu" and getattr(get_ops(), "name", "") == "sm90":  # (tests inject CPU chunk operators)
        if ctx.window is not None:
            raise NotImplementedError("window_size is not supported with host-resident (pinned CPU) operands; pass "
                                      "CUDA tensors")
        if ctx.alibi is not None:
            raise NotImplementedError("alibi_slopes is not supported with host-resident (pinned CPU) operands; pass "
                                      "CUDA tensors")
        # host-resident operands (pinned CPU tensors, one rank): copies stream under the kernels (host_stream.py)
        from . import host_stream
        if not host_stream.is_host_call(q, k, v):
            raise TypeError("burst_attn_b200 needs CUDA tensors (or pinned CPU tensors on a CUDA machine); there is "
                            "no CPU implementation")
        assert ctx.topo.W == 1, "host-resident operands are supported on a single rank only (pass device tensors)"
        assert q.shape[-1] in getattr(get_ops(), "tile_head_dims", (q.shape[-1],)), "host-resident operands need head_dim 64 or 128"
        ctx.host, ctx.mode, ctx.head_dim = True, mode, q.shape[-1]
        o_host, saved = host_stream.forward(q, k, v, ctx.softmax_scale, ctx.seq_dim, mode != "none", _l2_block())
        ctx.save_for_backward(*saved)
        return o_host
    (qp, kp, vp), ctx.head_dim = _pad_head_dim(get_ops(), [q, k, v])
    out, lse = _ring_forward(qp, kp, vp, ctx.softmax_scale, ctx.seq_dim, mode, ctx.topo, ctx.window, layout, ctx.alibi)
    ctx.mode, ctx.layout = mode, layout
    ctx.save_for_backward(qp, kp, vp, lse, out)
    return _unpad(out, ctx.head_dim)


def _op_backward(ctx, grad_output):
    if ctx.host:
        from . import host_stream
        grads = host_stream.backward(grad_output, ctx.saved_tensors, ctx.softmax_scale, ctx.seq_dim,
                                     ctx.mode != "none", _l2_block(), ctx.deterministic)
        return tuple(grads) + (None,) * 9
    q, k, v, lse, out = ctx.saved_tensors
    (g,), _ = _pad_head_dim(get_ops(), [grad_output])
    dq, dk, dv = _ring_backward(g, q, k, v, out, lse, ctx.softmax_scale, ctx.seq_dim, ctx.mode, ctx.topo,
                                ctx.deterministic, ctx.window, ctx.layout, ctx.alibi)
    return tuple(_unpad(t, ctx.head_dim) for t in (dq, dk, dv)) + (None,) * 9


class OpBurstAttn(torch.autograd.Function):
    """
    for Normal Attention (flash=None):  q, k, v: [B, N, S, H]
    for Flash ("cuda"/"triton"):        q, k, v: [B, S, N, H]
    Each rank passes its own sequence shard: contiguous when non-causal, zigzag
    halves {i, 2W-1-i} when causal.  window_size: flash-attn's (left, right) sliding window over positions of
    the full sequence (-1: unlimited side; causal forces right = 0).  alibi_slopes: flash-attn's ALiBi, fp32
    (nheads,) or (batch, nheads) per query head: the bias -slope |pos_q - pos_k| over the same positions.
    """

    @staticmethod
    def forward(ctx, q, k, v, softmax_scale=None, flash="cuda", causal=False, optimize_bwd_comm=False,
                deterministic=False, process_group=None, double_group=[None, None], window_size=(-1, -1),
                alibi_slopes=None):
        _prepare(ctx, q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic, process_group,
                 double_group, window_size, alibi_slopes)
        return _op_forward(ctx, q, k, v, "zigzag" if causal else "none", "zigzag" if causal else "contiguous")

    @staticmethod
    def backward(ctx, grad_output):
        return _op_backward(ctx, grad_output)


class OpBurstAttnStrip(torch.autograd.Function):
    """Striped-causal variant: rank i owns tokens {i, i+W, i+2W, ...} (with or without causal; a window then
    counts positions of the full sequence as in OpBurstAttn)."""

    @staticmethod
    def forward(ctx, q, k, v, softmax_scale=None, flash="cuda", causal=False, optimize_bwd_comm=False,
                deterministic=False, process_group=None, double_group=[None, None], window_size=(-1, -1),
                alibi_slopes=None):
        _prepare(ctx, q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic, process_group,
                 double_group, window_size, alibi_slopes)
        return _op_forward(ctx, q, k, v, "striped" if causal else "none", "striped")

    @staticmethod
    def backward(ctx, grad_output):
        return _op_backward(ctx, grad_output)


def burst_attn_func_striped(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float = None,
                            flash: str = "cuda", causal: bool = False, optimize_bwd_comm: bool = False,
                            deterministic: bool = False, process_group=None, double_group=[None, None],
                            window_size=(-1, -1), alibi_slopes=None):
    return OpBurstAttnStrip.apply(q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic,
                                  process_group, double_group, window_size, alibi_slopes)


def burst_attn_func(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float = None,
                    flash: str = "cuda", causal: bool = False, optimize_bwd_comm: bool = False,
                    deterministic: bool = False, process_group=None, double_group=[None, None],
                    window_size=(-1, -1), alibi_slopes=None):
    return OpBurstAttn.apply(q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic,
                             process_group, double_group, window_size, alibi_slopes)
