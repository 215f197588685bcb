"""Generate golden vectors by RUNNING THE REFERENCE (a checkout of
MayDomine/Burst-Attention) on CPU.  The reference is not a dependency of this
project, so its outputs are committed as small .npz fixtures next to this
script; tests/test_oracle_golden.py pins oracle/attention_oracle.py to them.

The reference imports `bmtrain` (absent here) at module scope
(burst_attn_interface.py:1, comm.py:2-5); a stub module is injected -- no
reference source is modified or copied.

Run:  python tests/golden/make_golden.py <path of the reference checkout>
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _stub_bmtrain():
    bmt = types.ModuleType("bmtrain")
    bmt.init = types.SimpleNamespace(is_initialized=lambda: False)
    bmt.config = {}
    bmt.print_rank = print
    sys.modules["bmtrain"] = bmt
    d = types.ModuleType("bmtrain.distributed"); sys.modules["bmtrain.distributed"] = d
    ops = types.ModuleType("bmtrain.distributed.ops"); ops.ncclSend = ops.ncclRecv = None
    sys.modules["bmtrain.distributed.ops"] = ops
    nccl = types.ModuleType("bmtrain.nccl")
    for n in ("commCount", "groupEnd", "groupStart", "allReduce", "commRank"):
        setattr(nccl, n, None)
    sys.modules["bmtrain.nccl"] = nccl
    bmt.distributed, bmt.nccl = d, nccl


def ring_vectors(bu):
    """The reference's device-agnostic chunk path (inter_normal_attn / _backward, burst_utils.py:42-100) over a ring
    of W ranks simulated in one process, schedule of OpBurstAttn.forward/backward (burst_attn_interface.py:214-248,
    291-396) without the transport; layout [B,H,S,D], fp32.  Inputs are fp16-representable (stored losslessly as
    fp16); the outputs are stored at a fixed, seeded sample of 512 positions per tensor."""
    g = torch.Generator().manual_seed(0)
    B, H, S, D = 1, 1, 64, 32
    q, k, v, do = (torch.randn(B, H, S, D, generator=g).half().float() for _ in range(4))
    idx = torch.randperm(B * H * S * D, generator=g)[:512].sort().values
    out = dict(ring_q=q.half(), ring_k=k.half(), ring_v=v.half(), ring_do=do.half(), ring_idx=idx,
               ring_scale=torch.tensor(D ** -0.5))
    for W in (1, 4):
        qs, ks, vs, dos = (t.chunk(W, dim=2) for t in (q, k, v, do))
        outs, lses = [], []
        for i in range(W):
            m_i = lse_i = acc_o = None
            for r in range(W):  # round r: rank i holds the K/V shard of rank (i - r) mod W
                j = (i - r) % W
                acc_o, m_i, lse_i = bu.inter_normal_attn(qs[i], ks[j], vs[j], m_i, lse_i, acc_o, D ** -0.5, None)
            outs.append(acc_o * torch.exp(m_i - lse_i))
            lses.append(lse_i)
        dqs = [torch.zeros_like(t) for t in qs]
        dks = [torch.zeros_like(t) for t in ks]
        dvs = [torch.zeros_like(t) for t in vs]
        deltas = [(outs[i] * dos[i]).sum(-1, keepdim=True) for i in range(W)]
        for j in range(W):  # K/V at home on rank j, the Q-bundle of rank i visits
            for r in range(W):
                i = (j - r) % W
                buf = torch.empty_like(qs[i])
                bu.inter_normal_attn_backward(dos[i], qs[i], ks[j], vs[j], deltas[i], lses[i], buf, dks[j], dvs[j],
                                              D ** -0.5, None)
                dqs[i] += buf
        for name, parts in (("o", outs), ("dq", dqs), ("dk", dks), ("dv", dvs)):
            out[f"ring_W{W}_{name}"] = torch.cat(parts, dim=2).reshape(-1)[idx]
    np.savez_compressed(os.path.join(HERE, "reference_ring.npz"), **{k_: v_.numpy() for k_, v_ in out.items()})


def main(ref):
    _stub_bmtrain()
    sys.path.insert(0, ref)
    import burst_attn.burst_utils as bu
    import burst_attn.burst_attn_interface as bi

    ring_vectors(bu)

    torch.manual_seed(20260922)
    out = {}

    # ---- 1. chunked forward chain through inter_normal_attn (burst_utils.py:42-74)
    B, H, S, D, W = 1, 1, 64, 32, 4
    scale = 1.0 / D ** 0.5
    q = torch.randn(B, H, S, D)
    k = torch.randn(B, H, S, D)
    v = torch.randn(B, H, S, D)
    m_i = lse_i = acc_o = None
    for c in range(W):
        ks = k.chunk(W, dim=2)[c]
        vs = v.chunk(W, dim=2)[c]
        acc_o, m_i, lse_i = bu.inter_normal_attn(q, ks, vs, m_i, lse_i, acc_o, scale, None)
    o_final = acc_o * torch.exp(m_i - lse_i)  # burst_attn_interface.py:246-248
    out.update(fwd_q=q, fwd_k=k, fwd_v=v, fwd_acc_o=acc_o, fwd_m=m_i, fwd_lse=lse_i,
               fwd_o=o_final, fwd_W=torch.tensor(W), fwd_scale=torch.tensor(scale))

    # ---- 2. chunk backward through inter_normal_attn_backward (burst_utils.py:77-100)
    do = torch.randn(B, H, S, D)
    delta = (o_final * do).sum(-1, keepdim=True)
    dq_tot = torch.zeros_like(q)
    dk_parts, dv_parts = [], []
    for c in range(W):
        ks = k.chunk(W, dim=2)[c]
        vs = v.chunk(W, dim=2)[c]
        dq = torch.empty_like(q)
        dk = torch.zeros_like(ks)
        dv = torch.zeros_like(vs)
        bu.inter_normal_attn_backward(do, q, ks, vs, delta, lse_i, dq, dk, dv, scale, None)
        dq_tot += dq
        dk_parts.append(dk)
        dv_parts.append(dv)
    out.update(bwd_do=do, bwd_delta=delta, bwd_dq=dq_tot,
               bwd_dk=torch.cat(dk_parts, 2), bwd_dv=torch.cat(dv_parts, 2))

    # ---- 3. LSE merge cuda_scale_out_lse_helper (burst_utils.py:20-33)
    Bm, Sm, Hm, Dm = 1, 16, 2, 8
    o = torch.randn(Bm, Sm, Hm, Dm)
    lse = torch.randn(Bm, Sm, Hm, 1) * 3
    o_new = torch.randn(Bm, Sm, Hm, Dm)
    lse_new = torch.randn(Bm, Hm, Sm) * 3
    mo, ml = bu.cuda_scale_out_lse_helper(o, lse, o_new, lse_new)
    out.update(merge_o=o, merge_lse=lse, merge_o_i=o_new, merge_lse_i=lse_new,
               merge_out_o=mo, merge_out_lse=ml)

    # ---- 4. get_partition_id (burst_attn_interface.py:20-37) single + double ring
    L, M = 4, 2  # 2 "nodes" of 4 (test/test_burst.py:129-138)
    table = np.zeros((L * M, L * M), dtype=np.int64)  # [rank, r-1]
    single = np.array([bi.get_partition_id([None, None], r) if False else r - 1
                       for r in range(1, L * M + 1)], dtype=np.int64)
    saved = (bi.get_rank, bi.get_world_size)
    try:
        for rank in range(L * M):
            intra, inter = rank % L, rank // L
            bi.get_rank = lambda g=None: {"intra": intra, "inter": inter}.get(g, rank)
            bi.get_world_size = lambda g=None: {"intra": L, "inter": M}.get(g, L * M)
            for r in range(1, L * M + 1):
                table[rank, r - 1] = bi.get_partition_id(("intra", "inter"), r)
        # single ring through the real function
        bi.get_rank = lambda g=None: 0
        bi.get_world_size = lambda g=None: L * M
        single = np.array([bi.get_partition_id([None, None], r) for r in range(1, L * M + 1)],
                          dtype=np.int64)
    finally:
        bi.get_rank, bi.get_world_size = saved
    out.update(pid_double=torch.from_numpy(table), pid_single=torch.from_numpy(single),
               pid_L=torch.tensor(L), pid_M=torch.tensor(M))

    # ---- 5. whole-op forward on CPU, W=1, flash=None ("normal" path, [B,H,S,D])
    try:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29577")
        dist.init_process_group("gloo", rank=0, world_size=1)
        qq = torch.randn(1, 1, 32, 16)
        kk = torch.randn(1, 1, 32, 16)
        vv = torch.randn(1, 1, 32, 16)
        oo = bi.burst_attn_func(qq, kk, vv, None, None, False)
        out.update(op_q=qq, op_k=kk, op_v=vv, op_o=oo)
        dist.destroy_process_group()
    except Exception as e:  # pragma: no cover - recorded in the fixture
        print("whole-op CPU forward not runnable:", repr(e))

    np.savez_compressed(os.path.join(HERE, "reference_vectors.npz"),
                        **{k_: v_.detach().cpu().numpy() for k_, v_ in out.items()})
    print("wrote", os.path.join(HERE, "reference_vectors.npz"), sorted(out))


if __name__ == "__main__":
    main(sys.argv[1])
