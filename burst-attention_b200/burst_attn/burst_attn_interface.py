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

import bisect
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


# --------------------------------------------------------------------------- #
# launch planning: every call is a band of key positions around each query position
# --------------------------------------------------------------------------- #
def _check_window(window_size, causal):
    """flash-attn's ``window_size=(left, right)`` (-1 or None: unlimited; ``causal`` forces right = 0) -> the band
    ``(left, right)`` of the call, None for an unlimited side: key position c is visible to query position a iff
    a - left <= c <= a + right."""
    if window_size is None:
        window_size = (-1, -1)
    try:
        left, right = (int(x) for x in window_size)
    except (TypeError, ValueError):
        raise ValueError(f"window_size must be a pair (left, right) of ints, got {window_size!r}") from None
    for name, x in (("left", left), ("right", right)):
        if x < -1:
            raise ValueError(f"window_size: {name} = {x}; it must be -1 (unlimited) or >= 0")
    return None if left == -1 else left, 0 if causal else (None if right == -1 else right)


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


def _sub(piece, r0, rn, c0, cn):
    """Rows [r0, r0+rn) and keys [c0, c0+cn) of a piece (local to it) as a launch of their own, or None when none of
    those rows sees any of those keys."""
    qa, _, ka, _, lo, hi = piece
    b = _band(rn, cn, None if lo is None else lo + r0 - c0, None if hi is None else hi + r0 - c0) \
        if rn > 0 and cn > 0 else None
    return None if b is None else (qa + r0, rn, ka + c0, cn) + b


def _merged(pieces):
    """A round's pieces as one launch over their bounding box when one band reproduces every sub-block exactly (so
    zigzag's own round, and its j < i and j > i rounds, are one launch each), else as they are.  Each side of the box
    band is taken from the first piece bounded on it: a side that binds in a piece is that piece's side exactly."""
    if len(pieces) < 2:
        return pieces
    rows, keys = sorted({p[:2] for p in pieces}), sorted({p[2:4] for p in pieces})
    q0, k0 = rows[0][0], keys[0][0]
    qn, kn = sum(n for _, n in rows), sum(n for _, n in keys)
    side = lambda s: next((p[s] - (p[0] - q0) + (p[2] - k0) for p in pieces if p[s] is not None), None)  # noqa: E731
    box = (q0, qn, k0, kn, side(4), side(5))
    have = {p[:4]: p for p in pieces}
    if any(_sub(box, qa - q0, rn, ka - k0, cn) != have.get((qa, rn, ka, cn)) for qa, rn in rows for ka, cn in keys):
        return pieces
    return [_sub(box, 0, qn, 0, kn)]


def _round_pieces(layout, W, iq, jk, Sq, Sk, band, merge=True, cu=None):
    """The pieces of the round that attends the Q shard of rank ``iq`` (``Sq`` rows) to the K/V shard of rank ``jk``
    (``Sk`` keys): ``[(q0, qn, k0, kn, lo, hi)]``, rows and keys local to the shards, the band relative to the two
    views; pieces whose band misses its view are left out, and with ``merge`` exact merges are made (``_merged``).
    ``cu``: the host list of document boundaries (``_check_cu_seqlens``), or None; each piece is then trimmed to the
    rows and keys that share a document (``_doc_trim``), and a piece whose rows share none with its keys is left out.
    ``band`` = (left, right) counts positions in the full sequence: contiguous shards start at rank * S, zigzag shards
    are the halves rank and 2W-1-rank (one piece per pair of halves), and striped token a of rank r sits at a W + r,
    so a + ceil((iq-jk-left)/W) <= c <= a + floor((iq-jk+right)/W)."""
    left, right = band
    if layout == "striped":
        cand = [(0, Sq, 0, Sk, None if left is None else -((jk - iq + left) // W),
                 None if right is None else (iq - jk + right) // W)]
    else:
        if layout == "contiguous":
            qs, ks = [(0, Sq, iq * Sq)], [(0, Sk, jk * Sk)]
        else:
            assert Sq % 2 == 0 and Sk % 2 == 0, "zigzag causal sharding needs an even local sequence length"
            h = Sq // 2
            qs = [(0, h, iq * h), (h, h, (2 * W - 1 - iq) * h)]
            ks = [(0, h, jk * h), (h, h, (2 * W - 1 - jk) * h)]
        cand = [(qa, qn, ka, kn, None if left is None else qg - kg - left, None if right is None else qg - kg + right)
                for qa, qn, qg in qs for ka, kn, kg in ks]
    out = [p for p in (_sub(c, 0, c[1], 0, c[3]) for c in cand) if p is not None]
    if cu is not None:
        pos_q, pstride = _positions(layout, W, iq, Sq)
        pos_k, _ = _positions(layout, W, jk, Sk)
        out = [p for p in (_doc_trim(p, cu, pos_q, pos_k, pstride) for p in out) if p is not None]
    return _merged(out) if merge else out


def _doc_of(cu, x):
    """The document of position x: the last d with cu[d] <= x (zero-length documents skipped), in [0, n_docs)."""
    return bisect.bisect_right(cu, x, 0, len(cu) - 1) - 1


def _doc_trim(piece, cu, pos_q, pos_k, pstride):
    """A piece cut to its rows and keys in the documents both reach, or None when they share none.  Inside a piece
    positions are affine (``pos(x0 + x) = pos(x0) + pstride x``), so the documents of its rows run from that of its first
    row to that of its last (the same for keys), and the rows (keys) of a run of documents are one interval."""
    qa, qn, ka, kn = piece[:4]
    q0, k0 = pos_q(qa), pos_k(ka)
    d0 = max(_doc_of(cu, q0), _doc_of(cu, k0))
    d1 = min(_doc_of(cu, q0 + pstride * (qn - 1)), _doc_of(cu, k0 + pstride * (kn - 1)))
    if d0 > d1:
        return None
    at = lambda p0, n, x: min(n, max(0, -((p0 - x) // pstride)))  # noqa: E731  first index at or after position x
    r0, r1 = at(q0, qn, cu[d0]), at(q0, qn, cu[d1 + 1])
    c0, c1 = at(k0, kn, cu[d0]), at(k0, kn, cu[d1 + 1])
    return _sub(piece, r0, r1 - r0, c0, c1 - c0)


def _fwd_block(piece, c0, cn):
    """Keys [c0, c0+cn) of a piece with only the rows that see them, the first row kept on a multiple of 256 (a
    pair of 128-row tiles), or None."""
    qn, lo, hi = piece[1], piece[4], piece[5]
    r0 = 0 if hi is None else max(0, (c0 - hi) // 256 * 256)
    r1 = qn if lo is None else min(qn, c0 + cn - lo)
    return _sub(piece, r0, r1 - r0, c0, cn)


def _bwd_block(piece, r0, rn):
    """Rows [r0, r0+rn) of a piece with only the keys they see, or None."""
    kn, lo, hi = piece[3], piece[4], piece[5]
    c0 = 0 if lo is None else max(0, r0 + lo)
    c1 = kn if hi is None else min(kn, r0 + rn + hi)
    return _sub(piece, r0, rn, c0, c1 - c0)


def _fwd_band_launches(pieces):
    """Forward launches ``[(q0, qn, k0, kn, lo, hi)]`` of a round's pieces: a piece longer than 1.5 L2 blocks is
    split over blocks of keys (each launch carries the state; the state pass costs 2 x 512 B per row and head, the
    block > 8 MB of math)."""
    blk = _l2_block()
    out = []
    for p in pieces:
        if p[3] <= blk + blk // 2:
            out.append(p)
        else:
            out += [x for x in (_fwd_block(p, c0, min(blk, p[3] - c0)) for c0 in range(0, p[3], blk)) if x]
    return out


def _bwd_band_launches(pieces):
    """Backward launches of a round's pieces: a piece with more than 1.5 L2 blocks of rows is split over blocks of
    rows."""
    blk = _l2_block()
    out = []
    for p in pieces:
        if p[1] <= blk + blk // 2:
            out.append(p)
        else:
            out += [x for x in (_bwd_block(p, r0, min(blk, p[1] - r0)) for r0 in range(0, p[1], blk)) if x]
    return out


def _lower_kw(lo):
    """Keyword for the chunk operators: the band's lower edge (nothing without one)."""
    return {} if lo is None else {"lower": lo}


# --------------------------------------------------------------------------- #
# packed documents: flash-attn's cu_seqlens over positions of the full sequence
# --------------------------------------------------------------------------- #
def _check_cu_seqlens(cu_seqlens, S, device, name="cu_seqlens"):
    """flash-attn's document boundaries (int32, 1-D, ``(n_docs + 1,)``, ``[0] == 0``, non-decreasing, ``[-1] == S``,
    the length of the full sequence; repeated values are zero-length documents) -> ``(host list, device int32
    tensor)``, or None.  The host list plans the launches and the device copy is what the kernels read; a CUDA tensor
    costs one device-to-host copy (and synchronisation) per call, a CPU tensor one host-to-device copy."""
    if cu_seqlens is None:
        return None
    if not isinstance(cu_seqlens, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(cu_seqlens).__name__}")
    if cu_seqlens.dtype != torch.int32:
        raise TypeError(f"{name} must be int32, got {cu_seqlens.dtype}")
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2:
        raise ValueError(f"{name} must be 1-D with at least 2 entries (n_docs + 1), got shape {tuple(cu_seqlens.shape)}")
    cu = cu_seqlens.tolist()
    if cu[0] != 0 or cu[-1] != S:
        raise ValueError(f"{name} must start at 0 and end at the sequence length {S}, got {cu[0]} .. {cu[-1]}")
    if any(b < a for a, b in zip(cu, cu[1:])):
        raise ValueError(f"{name} must be non-decreasing")
    return cu, cu_seqlens.detach().to(device).contiguous()


def _ring_doc(docs, layout, W, iq, jk, Sq, Sk):
    """The documents of the round that attends the Q shard of rank iq to the K/V shard of rank jk: (device
    boundaries, n_docs, pos_q, pos_k, pstride) with the position functions of ``_positions``, or None."""
    if docs is None:
        return None
    pos_q, pstride = _positions(layout, W, iq, Sq)
    pos_k, _ = _positions(layout, W, jk, Sk)
    return docs[1], len(docs[0]) - 1, pos_q, pos_k, pstride


def _doc_kw(doc, q0, k0):
    """Keyword for the chunk operators: the documents of the launch whose rows start at local row q0 and keys at
    local key k0 (nothing without documents)."""
    if doc is None:
        return {}
    cu, n_docs, pos_q, pos_k, pstride = doc
    return {"doc": (cu, n_docs, pos_q(q0), pos_k(k0), pstride)}


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


def _ring_alibi(slopes, layout, W, iq, jk, S):
    """The ALiBi of the round that attends the Q shard of rank iq to the K/V shard of rank jk (or None)."""
    if slopes is None:
        return None
    pos_q, pstride = _positions(layout, W, iq, S)
    pos_k, _ = _positions(layout, W, jk, S)
    return slopes, pos_q, pos_k, pstride


class _BandForward:
    """The forward launches of a call, known up front for every round, and their first / last duties.  The state is
    started by the first launch only if it covers every row (otherwise it starts as O = 0, lse = -inf in memory); the
    last launch writes its own rows in 16 bit, and ``finish`` casts the other rows from the fp32 state."""

    def __init__(self, rounds, q, lse, S):
        flat = [x for launches in rounds for x in launches]
        self.first = bool(flat) and flat[0][0] == 0 and flat[0][1] == S
        self.last_rows = flat[-1][:2] if flat else (0, 0)
        self.n, self.done = len(flat), 0
        self.o_acc = None
        if not (self.n == 1 and self.first):
            self.o_acc = torch.empty(q.shape, dtype=torch.float32, device=q.device)
        if not self.first:
            self.o_acc.zero_()
            lse.fill_(float("-inf"))

    def run(self, ops, launches, q, k, v, lse, out, scale, seq_dim, bias=None, alibi=None, doc=None):
        for q0, qn, k0, kn, lo, hi in launches:
            first = self.first and self.done == 0
            last = self.done == self.n - 1
            rows = lambda t: t.narrow(seq_dim, q0, qn)  # noqa: E731
            ops.fwd_chunk(rows(q), k.narrow(seq_dim, k0, kn), v.narrow(seq_dim, k0, kn),
                          None if self.o_acc is None else rows(self.o_acc), lse.narrow(2, q0, qn),
                          rows(out) if last else None, scale, hi is not None, 0 if hi is None else hi, first, last,
                          seq_dim, **_bias_kw(bias, k0, kn), **_lower_kw(lo), **_alibi_kw(alibi, q0, k0),
                          **_doc_kw(doc, q0, k0))
            self.done += 1

    def finish(self, ops, out, seq_dim):
        q0, qn = self.last_rows
        for r0, rn in ((0, q0), (q0 + qn, out.shape[seq_dim] - q0 - qn)):
            if rn > 0:
                ops.cast(self.o_acc.narrow(seq_dim, r0, rn), out.narrow(seq_dim, r0, rn), seq_dim)


def _bwd_band_run(ops, launches, g, q, k, v, delta, lse, dq_part, dk_acc, dv_acc, scale, seq_dim, deterministic,
                  bias=None, alibi=None, doc=None):
    for q0, qn, k0, kn, lo, hi in launches:
        rows = lambda t: t.narrow(seq_dim, q0, qn)  # noqa: E731
        keys = lambda t: t.narrow(seq_dim, k0, kn)  # noqa: E731
        ops.bwd_chunk(rows(g), rows(q), keys(k), keys(v), delta.narrow(2, q0, qn), lse.narrow(2, q0, qn),
                      rows(dq_part), keys(dk_acc), keys(dv_acc), scale, hi is not None, 0 if hi is None else hi, seq_dim,
                      deterministic, **_bias_kw(bias, k0, kn), **_lower_kw(lo), **_alibi_kw(alibi, q0, k0),
                      **_doc_kw(doc, q0, k0))


def _check_inputs(q, k, v, seq_dim):
    assert q.dim() == 4 and k.shape == v.shape and q.shape[0] == k.shape[0] and q.shape[3] == k.shape[3], \
        "q, k, v must be 4-D with matching batch and head_dim"
    hq, hkv = q.shape[3 - seq_dim], k.shape[3 - seq_dim]
    assert hkv > 0 and hq % hkv == 0, \
        f"the number of q heads ({hq}) must be a multiple of the number of k/v heads ({hkv})"
    assert q.dtype == k.dtype == v.dtype, "q, k, v must share a dtype"


# --------------------------------------------------------------------------- #
# forward ring (reference OpBurstAttn.forward :171-253, OpBurstAttnStrip.forward :411-493)
# --------------------------------------------------------------------------- #
def _ring_forward(q, k, v, scale, seq_dim, layout, band, topo, alibi=None, docs=None):
    """layout: the shards ("contiguous" | "zigzag" | "striped"); band: the call's (left, right) from
    ``_check_window``.  Returns (out, lse[B,H,S] fp32).  Each round runs the launches of ``_round_pieces``: the
    reference's zigzag rounds (plain causal own shard :221-224, all Q x first half of K/V :225-231, second half of Q x
    all K/V :232-235) and striped rounds (strictly lower triangular from a source rank ahead, :454,:463-475) are the
    pieces of the causal band.

    Rounds run in M cycles of L steps (the flat ring is one cycle, L = W).  Within a cycle K/V hop round the
    intra-node ring; on the hierarchical ring (reference comm.py:187-254, SURVEY.md Appendix C) the block a
    cycle starts with is at the same time forwarded to the next node over the inter-node ring, where it starts
    the following cycle -- a prefetch with L rounds of kernel time to hide behind.  Unlike the reference no
    send-side copy is made: the cycle's starting block is never a receive target while it is in flight (two
    inter-node buffers alternate).

    ``alibi`` (fp32 slopes [B, H] from ``_check_alibi``) gives every launch where its rows and keys sit in the full
    sequence; its pieces are not merged, since zigzag positions are not affine across the two halves.  ``docs``
    (``_check_cu_seqlens``) does the same for packed documents, and trims every piece to its shared documents."""
    ops = get_ops()
    ring, inter, _ = topo.rings()
    L, M, W, i = topo.L, topo.M, topo.W, topo.rank
    B, S, H = q.shape[0], q.shape[seq_dim], q.shape[3 - seq_dim]
    out = torch.empty_like(q)
    lse = torch.empty((B, H, S), dtype=torch.float32, device=q.device)
    Sk = k.shape[seq_dim]
    cu = None if docs is None else docs[0]
    plan = [_fwd_band_launches(_round_pieces(layout, W, i, topo.source(r), S, Sk, band,
                                             alibi is None and docs is None, cu))
            for r in range(1, W + 1)]
    state = _BandForward(plan, q, lse, S)
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
            # a round whose shard lies outside every row's band launches nothing
            state.run(ops, plan[r - 1], q, cur[0], cur[1], lse, out, scale, seq_dim,
                      alibi=_ring_alibi(alibi, layout, W, i, j, S), doc=_ring_doc(docs, layout, W, i, j, S, Sk))
            if t != L - 1:
                ring.wait()
                cur = nxt
            elif c != M - 1:
                inter.wait()
                cur = xbuf[c % len(xbuf)]
    state.finish(ops, out, seq_dim)
    return out, lse


# --------------------------------------------------------------------------- #
# backward ring (reference OpBurstAttn.backward :256-398, OpBurstAttnStrip.backward :496-613)
# --------------------------------------------------------------------------- #
def _ring_backward(d_o, q, k, v, out, lse, scale, seq_dim, layout, band, topo, deterministic, alibi=None, docs=None):
    """Backward of ``_ring_forward``: round r attends the Q-bundle of rank j = source(r) to the K/V at home."""
    ops = get_ops()
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
        dlt, g, qq, ls = bundle  # the bundle of rank j against the K/V at home: rows of j, keys of i
        Sk = k.shape[seq_dim]
        pieces = _round_pieces(layout, W, j, i, S, Sk, band, alibi is None and docs is None,
                               None if docs is None else docs[0])
        _bwd_band_run(ops, _bwd_band_launches(pieces), g, qq, k, v, dlt, ls, dq_part, dk_acc, dv_acc, scale, seq_dim,
                      deterministic, alibi=_ring_alibi(alibi, layout, W, j, i, S),
                      doc=_ring_doc(docs, layout, W, j, i, S, Sk))

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
             double_group, window_size=(-1, -1), alibi_slopes=None, cu_seqlens=None):
    assert not causal or flash == "cuda", "Causal attention only supported for Flash v2"
    ctx.band = _check_window(window_size, causal)
    ctx.alibi = _check_alibi(alibi_slopes, q, 2 if flash in ["cuda", "triton"] else 1)
    if cu_seqlens is not None and ctx.alibi is not None:
        raise NotImplementedError("cu_seqlens together with alibi_slopes is not supported")
    ctx.docs = None
    if cu_seqlens is not None:  # positions count the full sequence: W shards of the local length
        S = q.shape[1 if flash in ["cuda", "triton"] else 2] * get_world_size(process_group)
        ctx.docs = _check_cu_seqlens(cu_seqlens, S, q.device)
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


def _op_forward(ctx, q, k, v, layout):
    """layout: the call's shards ("contiguous" | "zigzag" | "striped")."""
    ctx.host, ctx.layout = False, layout
    if q.device.type == "cpu" and getattr(get_ops(), "name", "") == "sm90":  # (tests inject CPU chunk operators)
        if ctx.band != _check_window(None, ctx.causal):
            raise NotImplementedError("window_size is not supported with host-resident (pinned CPU) operands; pass "
                                      "CUDA tensors")
        if ctx.alibi is not None:
            raise NotImplementedError("alibi_slopes is not supported with host-resident (pinned CPU) operands; pass "
                                      "CUDA tensors")
        if ctx.docs is not None:
            raise NotImplementedError("cu_seqlens is not supported with host-resident (pinned CPU) operands; pass "
                                      "CUDA tensors")
        # host-resident operands (pinned CPU tensors, one rank): copies stream under the kernels (host_stream.py)
        from . import host_stream
        if not host_stream.is_host_call(q, k, v):
            raise TypeError("burst_attn_b200 needs CUDA tensors (or pinned CPU tensors on a CUDA machine); there is "
                            "no CPU implementation")
        assert ctx.topo.W == 1, "host-resident operands are supported on a single rank only (pass device tensors)"
        assert q.shape[-1] in getattr(get_ops(), "tile_head_dims", (q.shape[-1],)), "host-resident operands need head_dim 64 or 128"
        ctx.host, ctx.head_dim = True, q.shape[-1]
        o_host, saved = host_stream.forward(q, k, v, ctx.softmax_scale, ctx.seq_dim, ctx.band, _l2_block())
        ctx.save_for_backward(*saved)
        return o_host
    (qp, kp, vp), ctx.head_dim = _pad_head_dim(get_ops(), [q, k, v])
    out, lse = _ring_forward(qp, kp, vp, ctx.softmax_scale, ctx.seq_dim, layout, ctx.band, ctx.topo, ctx.alibi,
                             ctx.docs)
    ctx.save_for_backward(qp, kp, vp, lse, out)
    return _unpad(out, ctx.head_dim)


def _op_backward(ctx, grad_output):
    if ctx.host:
        from . import host_stream
        grads = host_stream.backward(grad_output, ctx.saved_tensors, ctx.softmax_scale, ctx.seq_dim, ctx.band,
                                     _l2_block(), ctx.deterministic)
        return tuple(grads) + (None,) * 10
    q, k, v, lse, out = ctx.saved_tensors
    (g,), _ = _pad_head_dim(get_ops(), [grad_output])
    dq, dk, dv = _ring_backward(g, q, k, v, out, lse, ctx.softmax_scale, ctx.seq_dim, ctx.layout, ctx.band, ctx.topo,
                                ctx.deterministic, ctx.alibi, ctx.docs)
    return tuple(_unpad(t, ctx.head_dim) for t in (dq, dk, dv)) + (None,) * 10


class OpBurstAttn(torch.autograd.Function):
    """
    for Normal Attention (flash=None):  q, k, v: [B, N, S, H]
    for Flash ("cuda"/"triton"):        q, k, v: [B, S, N, H]
    Each rank passes its own sequence shard: contiguous when non-causal, zigzag
    halves {i, 2W-1-i} when causal.  window_size: flash-attn's (left, right) sliding window over positions of
    the full sequence (-1: unlimited side; causal forces right = 0).  alibi_slopes: flash-attn's ALiBi, fp32
    (nheads,) or (batch, nheads) per query head: the bias -slope |pos_q - pos_k| over the same positions.
    cu_seqlens: flash-attn's packed-document boundaries over the same positions (int32, ``(n_docs + 1,)``, from 0 to
    the full sequence length, the same for every batch entry): a query sees only keys of its own document, on top of
    causal / window_size.  Not combined with alibi_slopes (``_check_cu_seqlens`` says what it costs).
    """

    @staticmethod
    def forward(ctx, q, k, v, softmax_scale=None, flash="cuda", causal=False, optimize_bwd_comm=False,
                deterministic=False, process_group=None, double_group=[None, None], window_size=(-1, -1),
                alibi_slopes=None, cu_seqlens=None):
        _prepare(ctx, q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic, process_group,
                 double_group, window_size, alibi_slopes, cu_seqlens)
        return _op_forward(ctx, q, k, v, "zigzag" if causal else "contiguous")

    @staticmethod
    def backward(ctx, grad_output):
        return _op_backward(ctx, grad_output)


class OpBurstAttnStrip(torch.autograd.Function):
    """Striped-causal variant: rank i owns tokens {i, i+W, i+2W, ...} (with or without causal; a window then
    counts positions of the full sequence as in OpBurstAttn)."""

    @staticmethod
    def forward(ctx, q, k, v, softmax_scale=None, flash="cuda", causal=False, optimize_bwd_comm=False,
                deterministic=False, process_group=None, double_group=[None, None], window_size=(-1, -1),
                alibi_slopes=None, cu_seqlens=None):
        _prepare(ctx, q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic, process_group,
                 double_group, window_size, alibi_slopes, cu_seqlens)
        return _op_forward(ctx, q, k, v, "striped")

    @staticmethod
    def backward(ctx, grad_output):
        return _op_backward(ctx, grad_output)


def burst_attn_func_striped(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float = None,
                            flash: str = "cuda", causal: bool = False, optimize_bwd_comm: bool = False,
                            deterministic: bool = False, process_group=None, double_group=[None, None],
                            window_size=(-1, -1), alibi_slopes=None, cu_seqlens=None):
    return OpBurstAttnStrip.apply(q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic,
                                  process_group, double_group, window_size, alibi_slopes, cu_seqlens)


def burst_attn_func(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float = None,
                    flash: str = "cuda", causal: bool = False, optimize_bwd_comm: bool = False,
                    deterministic: bool = False, process_group=None, double_group=[None, None],
                    window_size=(-1, -1), alibi_slopes=None, cu_seqlens=None):
    return OpBurstAttn.apply(q, k, v, softmax_scale, flash, causal, optimize_bwd_comm, deterministic,
                             process_group, double_group, window_size, alibi_slopes, cu_seqlens)
