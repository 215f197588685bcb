"""TEST-ONLY chunk operators backed by the CPU oracle, with the same five-method
interface as burst_attn.chunk_ops.NativeOps.  Injected with
``chunk_ops._set_ops_for_testing`` so the ring drivers (schedule, buffer
rotation, dQ ring, shard views) can be exercised under gloo with world_size > 1
on a machine without a GPU.  K/V may have fewer heads than Q (grouped-query attention,
query head h reads K/V head h // G): they are expanded per group before the oracle call and dK/dV are summed
back over each group.  The product never imports this."""
import torch

from oracle import attention_oracle as orc


def _bshd(t, seq_dim):
    return t if seq_dim == 1 else t.permute(0, 2, 1, 3)


def _expand(t, G):
    """[B,S,Hkv,D] -> [B,S,Hkv*G,D]: K/V head h // G for query head h."""
    return t if G == 1 else t.repeat_interleave(G, dim=2)


def _group_sum(t, G):
    """[B,S,Hkv*G,D] -> [B,S,Hkv,D]: the gradient of _expand."""
    return t if G == 1 else t.unflatten(2, (t.shape[2] // G, G)).sum(3)


def _mode(causal, off, sq, sk):
    if not causal:
        return "none"
    return ("causal_offset", off)


class OracleOps:
    name = "oracle(test)"

    def __init__(self):
        self.launches = 0
        self.calls = []

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None):
        self.calls.append(("fwd", tuple(q.shape), tuple(k.shape), causal, causal_offset, first, last))
        qq, kk, vv = (_bshd(t, seq_dim) for t in (q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = _mode(causal, causal_offset, qq.shape[1], kk.shape[1])
        st_o = None if first else _bshd(o_acc, seq_dim).double()
        st_l = None if first else lse.double()
        o, l = orc.chunk_forward(qq, kk, vv, st_o, st_l, scale, mode, key_bias=bias)
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
                  deterministic=False, bias=None):
        self.calls.append(("bwd", tuple(q.shape), tuple(k.shape), causal, causal_offset))
        g, qq, kk, vv = (_bshd(t, seq_dim) for t in (d_o, q, k, v))
        G = qq.shape[2] // kk.shape[2]
        kk, vv = _expand(kk, G), _expand(vv, G)
        mode = _mode(causal, causal_offset, qq.shape[1], kk.shape[1])
        ls = torch.where(torch.isinf(lse), torch.full_like(lse, 1e30), lse)
        dq, dk, dv = orc.chunk_backward(g, qq, kk, vv, delta, ls, scale, mode, key_bias=bias)
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
