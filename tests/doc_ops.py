"""TEST-ONLY chunk operators with packed documents: ``band_ops.BandOracleOps`` plus the ``doc`` keyword of
``burst_attn.chunk_ops.NativeOps`` (``(cu_seqlens, n_docs, q_pos0, k_pos0, pstride)``), so the document ring drivers
run under gloo on a machine without a GPU.  A call without ``doc`` is the plain ``BandOracleOps`` call.  Every doc call
is recorded in ``calls`` with its lower edge and ``(n_docs, q_pos0, k_pos0, pstride)`` appended, and the forward's
visible (row position, key position) pairs are collected in ``pairs`` (a pair seen twice is an error)."""
import torch

import band_oracle as bo
import doc_oracle as do_
from oracle_ops import _bshd, _expand, _group_sum
from band_ops import BandOracleOps


def launch_mask(sq, sk, causal, causal_offset, lower, doc):
    """The kernels' mask of one doc launch: band (lower edge, causal offset) and documents."""
    cu, n_docs, q_pos0, k_pos0, pstride = doc
    cu = [int(x) for x in cu.tolist()]
    assert len(cu) == n_docs + 1
    pq, pk = q_pos0 + pstride * torch.arange(sq), k_pos0 + pstride * torch.arange(sk)
    m = do_.same_doc(pq, pk, cu)
    b = bo.band_mask(sq, sk, ("band", lower, causal_offset if causal else None))
    return (m if b is None else m & b), pq, pk


class DocOracleOps(BandOracleOps):
    name = "oracle-doc(test)"

    def __init__(self):
        super().__init__()
        self.pairs = set()

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None, doc=None):
        if doc is None:
            return super().fwd_chunk(q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim,
                                     bias, lower)
        assert bias is None
        self.calls.append(("fwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, first, last, lower,
                           tuple(int(x) for x in doc[1:])))
        qq, kk, vv = (_bshd(t, seq_dim) for t in (q, k, v))
        kk, vv = _expand(kk, qq.shape[2] // kk.shape[2]), _expand(vv, qq.shape[2] // kk.shape[2])
        m, pq, pk = launch_mask(qq.shape[1], kk.shape[1], causal, causal_offset, lower, doc)
        for a, c in m.nonzero().tolist():
            pair = (int(pq[a]), int(pk[c]))
            assert pair not in self.pairs, f"pair {pair} attended twice"
            self.pairs.add(pair)
        st_o = None if first else _bshd(o_acc, seq_dim).double()
        st_l = None if first else lse.double()
        o, l = do_.masked_chunk_forward(qq, kk, vv, st_o, st_l, scale, m)
        lse.copy_(l.to(lse.dtype))
        if last:
            _bshd(o_out, seq_dim).copy_(o.to(o_out.dtype))
        else:
            _bshd(o_acc, seq_dim).copy_(o.to(o_acc.dtype))
        self.launches += 1

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None, doc=None):
        if doc is None:
            return super().bwd_chunk(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset,
                                     seq_dim, deterministic, bias, lower)
        assert bias is None
        self.calls.append(("bwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, lower,
                           tuple(int(x) for x in doc[1:])))
        g, qq, kk, vv = (_bshd(t, seq_dim) for t in (d_o, q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        m, _, _ = launch_mask(qq.shape[1], kk.shape[1], causal, causal_offset, lower, doc)
        ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
        dq, dk, dv = do_.masked_chunk_backward(g, qq, kk, vv, delta, ls, scale, m)
        _bshd(dq_acc, seq_dim).add_(dq.to(dq_acc.dtype))
        _bshd(dk_acc, seq_dim).add_(_group_sum(dk, G).to(dk_acc.dtype))
        _bshd(dv_acc, seq_dim).add_(_group_sum(dv, G).to(dv_acc.dtype))
        self.launches += 1
