"""TEST-ONLY chunk operators with a band mask: ``oracle_ops.OracleOps`` plus the ``lower`` keyword of
``burst_attn.chunk_ops.NativeOps`` (key c visible to row a only if c >= a + lower), so the windowed ring drivers can run
under gloo on a machine without a GPU.  A call without ``lower`` is the plain ``OracleOps`` call.  Every call is
recorded as in ``OracleOps.calls`` with the lower edge (or None) appended."""
import torch

import band_oracle as bo
from oracle_ops import OracleOps, _bshd, _expand, _group_sum


class BandOracleOps(OracleOps):
    name = "oracle-band(test)"

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None):
        if lower is None:
            super().fwd_chunk(q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias)
            self.calls[-1] += (None,)
            return
        self.calls.append(("fwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, first, last, lower))
        qq, kk, vv = (_bshd(t, seq_dim) for t in (q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = ("band", lower, causal_offset if causal else None)
        st_o = None if first else _bshd(o_acc, seq_dim).double()
        st_l = None if first else lse.double()
        o, l = bo.chunk_forward(qq, kk, vv, st_o, st_l, scale, mode, key_bias=bias)
        lse.copy_(l.to(lse.dtype))
        if last:
            _bshd(o_out, seq_dim).copy_(o.to(o_out.dtype))
        else:
            _bshd(o_acc, seq_dim).copy_(o.to(o_acc.dtype))
        self.launches += 1

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None):
        if lower is None:
            super().bwd_chunk(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                              deterministic, bias)
            self.calls[-1] += (None,)
            return
        self.calls.append(("bwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, lower))
        g, qq, kk, vv = (_bshd(t, seq_dim) for t in (d_o, q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = ("band", lower, causal_offset if causal else None)
        ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
        dq, dk, dv = bo.chunk_backward(g, qq, kk, vv, delta, ls, scale, mode, key_bias=bias)
        _bshd(dq_acc, seq_dim).add_(dq.to(dq_acc.dtype))
        _bshd(dk_acc, seq_dim).add_(_group_sum(dk, G).to(dk_acc.dtype))
        _bshd(dv_acc, seq_dim).add_(_group_sum(dv, G).to(dv_acc.dtype))
        self.launches += 1
