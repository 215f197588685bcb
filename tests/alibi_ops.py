"""TEST-ONLY chunk operators with ALiBi: ``band_ops.BandOracleOps`` plus the ``alibi`` keyword of
``burst_attn.chunk_ops.NativeOps`` (``(slopes [B, H], dist0, pstride)``), so the ALiBi ring drivers can run under gloo
on a machine without a GPU.  A call without ``alibi`` is the plain ``BandOracleOps`` call.  Every call is recorded as
in ``BandOracleOps.calls`` with ``(dist0, pstride)`` (or None) appended."""
import torch

import alibi_oracle as ao
from oracle_ops import _bshd, _expand, _group_sum
from band_ops import BandOracleOps


class AlibiOracleOps(BandOracleOps):
    name = "oracle-alibi(test)"

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None, alibi=None):
        if alibi is None:
            super().fwd_chunk(q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias,
                              lower)
            self.calls[-1] += (None,)
            return
        assert bias is None
        self.calls.append(("fwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, first, last, lower,
                           (int(alibi[1]), int(alibi[2]))))
        qq, kk, vv = (_bshd(t, seq_dim) for t in (q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = ("band", lower, causal_offset if causal else None)
        st_o = None if first else _bshd(o_acc, seq_dim).double()
        st_l = None if first else lse.double()
        o, l = ao.chunk_forward(qq, kk, vv, st_o, st_l, scale, mode, alibi)
        lse.copy_(l.to(lse.dtype))
        if last:
            _bshd(o_out, seq_dim).copy_(o.to(o_out.dtype))
        else:
            _bshd(o_acc, seq_dim).copy_(o.to(o_acc.dtype))
        self.launches += 1

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None, alibi=None):
        if alibi is None:
            super().bwd_chunk(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                              deterministic, bias, lower)
            self.calls[-1] += (None,)
            return
        assert bias is None
        self.calls.append(("bwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, lower,
                           (int(alibi[1]), int(alibi[2]))))
        g, qq, kk, vv = (_bshd(t, seq_dim) for t in (d_o, q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = ("band", lower, causal_offset if causal else None)
        ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
        dq, dk, dv = ao.chunk_backward(g, qq, kk, vv, delta, ls, scale, mode, alibi)
        _bshd(dq_acc, seq_dim).add_(dq.to(dq_acc.dtype))
        _bshd(dk_acc, seq_dim).add_(_group_sum(dk, G).to(dk_acc.dtype))
        _bshd(dv_acc, seq_dim).add_(_group_sum(dv, G).to(dv_acc.dtype))
        self.launches += 1
