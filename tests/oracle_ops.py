"""TEST-ONLY chunk operators backed by the fp64 CPU oracle (``mask_oracle``), with the interface of
burst_attn.chunk_ops.NativeOps: the same five methods and, on ``fwd_chunk`` / ``bwd_chunk``, the same keywords --
``bias`` (a key bias), ``lower`` (key c visible to row a only if c >= a + lower), ``alibi`` (``(slopes [B, H], dist0,
pstride)``) and ``doc`` (``(cu_seqlens, n_docs, q_pos0, k_pos0, pstride)``).  Injected with
``chunk_ops._set_ops_for_testing`` so the ring drivers (schedule, buffer rotation, dQ ring, shard views) can be
exercised under gloo with world_size > 1 on a machine without a GPU.  K/V may have fewer heads than Q (grouped-query
attention, query head h reads K/V head h // G): they are expanded per group before the oracle call and dK/dV are
summed back over each group.

Every chunk call is recorded in ``calls`` as a ``Call``; the forward's visible (row position, key position) pairs of
document calls are collected in ``pairs`` (a pair seen twice is an error).  The product never imports this."""
from collections import namedtuple

import torch

import mask_oracle as mo
from oracle import attention_oracle as orc

# kind "fwd" / "bwd"; first / last: None for "bwd"; alibi: (dist0, pstride); doc: (n_docs, q_pos0, k_pos0, pstride)
Call = namedtuple("Call", "kind q k causal causal_offset first last lower alibi doc")


def _bshd(t, seq_dim):
    return t if seq_dim == 1 else t.permute(0, 2, 1, 3)


def _expand(t, G):
    """[B,S,Hkv,D] -> [B,S,Hkv*G,D]: K/V head h // G for query head h."""
    return t if G == 1 else t.repeat_interleave(G, dim=2)


def _group_sum(t, G):
    """[B,S,Hkv*G,D] -> [B,S,Hkv,D]: the gradient of _expand."""
    return t if G == 1 else t.unflatten(2, (t.shape[2] // G, G)).sum(3)


def _mask(causal, causal_offset, lower, doc):
    """The kernels' mask of one call (``mask_oracle.mask_of``)."""
    hi = causal_offset if causal else None
    if doc is not None:
        cu, n_docs, q_pos0, k_pos0, pstride = doc
        cu = tuple(int(x) for x in cu.tolist())
        assert len(cu) == n_docs + 1
        return ("doc", lower, hi, cu, q_pos0, k_pos0, pstride)
    if lower is not None:
        return ("band", lower, hi)
    return ("causal_offset", causal_offset) if causal else None


def _call(kind, q, k, causal, causal_offset, first, last, lower, alibi, doc):
    return Call(kind, tuple(q.shape), tuple(k.shape), causal, causal_offset, first, last, lower,
                None if alibi is None else (int(alibi[1]), int(alibi[2])),
                None if doc is None else tuple(int(x) for x in doc[1:]))


class OracleOps:
    name = "oracle(test)"

    def __init__(self):
        self.launches = 0
        self.calls = []
        self.pairs = set()

    def _operands(self, q, k, v, seq_dim, bias, alibi):
        qq, kk, vv = (_bshd(t, seq_dim) for t in (q, k, v))
        G = qq.shape[2] // kk.shape[2]
        if alibi is not None:
            assert bias is None
            bias = mo.chunk_bias(alibi, qq.shape[1], kk.shape[1])
        return qq, _expand(kk, G), _expand(vv, G), G, bias

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None, alibi=None, doc=None):
        self.calls.append(_call("fwd", q, k, causal, causal_offset, first, last, lower, alibi, doc))
        qq, kk, vv, _, bias = self._operands(q, k, v, seq_dim, bias, alibi)
        mask = _mask(causal, causal_offset, lower, doc)
        if doc is not None:
            assert bias is None
            _, _, _, _, q_pos0, k_pos0, ps = mask
            for a, c in mo.mask_of(qq.shape[1], kk.shape[1], mask).nonzero().tolist():
                pair = (int(q_pos0 + ps * a), int(k_pos0 + ps * c))
                assert pair not in self.pairs, f"pair {pair} attended twice"
                self.pairs.add(pair)
        st_o = None if first else _bshd(o_acc, seq_dim).double()
        st_l = None if first else lse.double()
        o, l = mo.chunk_forward(qq, kk, vv, st_o, st_l, scale, mask, bias=bias)
        lse.copy_(l.to(lse.dtype))
        if last:
            _bshd(o_out, seq_dim).copy_(o.to(o_out.dtype))
        else:
            _bshd(o_acc, seq_dim).copy_(o.to(o_acc.dtype))
        self.launches += 1

    def delta(self, o, d_o, out, seq_dim):
        out.copy_(orc.compute_delta(_bshd(o, seq_dim), _bshd(d_o, seq_dim)).to(out.dtype))
        self.launches += 1

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None, alibi=None, doc=None):
        self.calls.append(_call("bwd", q, k, causal, causal_offset, None, None, lower, alibi, doc))
        qq, kk, vv, G, bias = self._operands(q, k, v, seq_dim, bias, alibi)
        g = _bshd(d_o, seq_dim)
        ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
        dq, dk, dv = mo.chunk_backward(g, qq, kk, vv, delta, ls, scale, _mask(causal, causal_offset, lower, doc),
                                       bias=bias)
        _bshd(dq_acc, seq_dim).add_(dq.to(dq_acc.dtype))
        _bshd(dk_acc, seq_dim).add_(_group_sum(dk, G).to(dk_acc.dtype))
        _bshd(dv_acc, seq_dim).add_(_group_sum(dv, G).to(dv_acc.dtype))
        self.launches += 1

    def cast(self, src, dst, seq_dim):
        dst.copy_(src.to(dst.dtype))
        self.launches += 1

    def accumulate(self, src, dst, seq_dim):
        dst.add_(src)
        self.launches += 1
