"""Record the kernel launch plans of the attention drivers and keep a summary of each in ``plans.json``: for each
configuration below, every chunk-operator call the ring drivers (``_ring_forward`` / ``_ring_backward``), the
single-GPU wrappers (``flash_attn_func``) and the host-resident path (``host_stream``) make, in order (``summary``
says what is kept).

No GPU and no memory are needed: operands are ``meta`` tensors, the chunk operators only record, the topology is a
stub of one rank of a flat ring and the ring moves nothing.  A launch is recorded as its row and key views (offset,
length), its mask (causal, causal_offset, lower), FIRST / LAST, the rows its LAST writes and its ALiBi distance;
``wait`` marks the end of a ring round.

    python tests/golden/make_plans.py [package dir] [output]

The fixture was recorded from the commit before the single launch planner (package ``burst-attention_b200`` of that
commit); ``tests/test_launch_plans.py`` compares the current drivers against it."""
import contextlib
import hashlib
import inspect
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def _configs():
    ring = lambda layout, causal, W, rank, S, **kw: dict(kind="ring", layout=layout, causal=causal, W=W, rank=rank,  # noqa: E731
                                                         S=S, **kw)
    out = []
    # the benchmark's workloads: one GPU at S = 65536, eight at 32768 per rank
    for causal, layout in ((False, "contiguous"), (True, "zigzag")):
        out.append(ring(layout, causal, 1, 0, 65536, H=32, D=128))
        out += [ring(layout, causal, 8, r, 32768, H=32, D=128) for r in range(8)]
    cases = [("contiguous", False), ("zigzag", True), ("striped", False), ("striped", True)]
    for layout, causal in cases:
        # tiny L2 blocks with ragged lengths
        for blk, S in ((8, 70), (16, 202), (24, 70), (100, 602), (256, 602)):
            out += [ring(layout, causal, W, r, S, blk=blk) for W in ((1, 2) if blk in (16, 100) else (1,))
                    for r in range(W)]
        # every rank of every ring size
        out += [ring(layout, causal, W, r, 64, blk=16) for W in (4, 8) for r in range(W)]
        # windows and ALiBi
        for extra in (dict(window=(5, 3)), dict(window=(40, 0)), dict(alibi=True), dict(alibi=True, window=(9, 9))):
            out += [ring(layout, causal, 4, r, 64, blk=16, **extra) for r in range(4)]
    # flash_attn_func, bottom-right aligned, Sq != Sk included
    for blk in (16, 256):
        for Sq, Sk in ((70, 70), (600, 40), (40, 600)) + (((1000, 3000), (3000, 1000)) if blk > 16 else ()):
            for causal in (False, True):
                for extra in ({}, dict(window=(64, 64)), dict(alibi=True)):
                    out.append(dict(kind="local", Sq=Sq, Sk=Sk, causal=causal, blk=blk, **extra))
    # host-resident operands
    for S, blk in ((600, 256), (602, 100), (65536, 32768), (65536, 16384)):
        out += [dict(kind="host", S=S, causal=causal, blk=blk) for causal in (False, True)]
    return out


CONFIGS = _configs()


def key(cfg):
    rest = [f"{k}={cfg[k]}".replace(" ", "") for k in sorted(cfg) if k not in ("kind", "layout", "causal", "alibi")]
    return " ".join([cfg["kind"], cfg.get("layout", ""), "causal" if cfg["causal"] else "full"] + rest
                    + (["alibi"] if cfg.get("alibi") else [])).replace("  ", " ")


def plain(cfg):
    """A call without window or ALiBi: its launches must not change."""
    return cfg.get("window", (-1, -1)) == (-1, -1) and not cfg.get("alibi")


def rows_of(cfg):
    return cfg["Sq"] if cfg["kind"] == "local" else cfg["S"]


def _rows(t, dim):
    """(offset, length) of a view along ``dim`` within its base tensor."""
    return [t.storage_offset() // t.stride(dim), t.shape[dim]]


class RecordingOps:
    """Chunk operators that do nothing but log their calls."""
    name = "recording"

    def __init__(self, log):
        self.log = log

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None,
                  lower=None, alibi=None):
        self.log.append(["fwd", _rows(q, seq_dim), _rows(k, seq_dim), bool(causal), int(causal_offset), lower,
                         bool(first), bool(last), None if o_out is None else _rows(o_out, seq_dim),
                         None if alibi is None else [int(alibi[1]), int(alibi[2])]])

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, bias=None, lower=None, alibi=None):
        self.log.append(["bwd", _rows(q, seq_dim), _rows(k, seq_dim), bool(causal), int(causal_offset), lower,
                         None if alibi is None else [int(alibi[1]), int(alibi[2])]])

    def cast(self, src, dst, seq_dim):
        self.log.append(["cast", _rows(dst, seq_dim)])

    def delta(self, o, d_o, out, seq_dim):
        pass

    def accumulate(self, src, dst, seq_dim):
        pass


class _Ring:
    def __init__(self, log):
        self.log = log

    def begin(self, *a):
        pass

    def post(self, *a):
        pass

    def wait(self):
        self.log.append(["wait"])

    def empty(self, shape, dtype, dev):
        return torch.empty(shape, dtype=dtype, device="meta")

    def empty_like(self, t):
        return torch.empty_like(t, device="meta")


class _Topology:
    """Rank ``rank`` of a flat ring of ``W``."""

    def __init__(self, W, rank, log):
        self.W, self.rank, self.L, self.M, self.log = W, rank, W, 1, log

    def source(self, r):
        return (self.rank - (r - 1)) % self.W

    def rings(self):
        return _Ring(self.log), None, None


class _Nothing:
    """A CUDA stream, event or stream context that does nothing."""

    def __init__(self, *a, **k):
        pass

    def __getattr__(self, name):
        return lambda *a, **k: None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


class _MetaTorch:
    """``torch`` as the host-resident path sees it while recording: streams and events do nothing, every tensor is on
    ``meta``."""

    class cuda:
        Stream = Event = _Nothing
        current_device = staticmethod(lambda: 0)
        current_stream = staticmethod(lambda dev=None: _Nothing())
        stream = staticmethod(lambda s: _Nothing())

    device = staticmethod(lambda *a: torch.device("meta"))

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def empty(*a, **k):
        k.pop("pin_memory", None)
        return torch.empty(*a, **dict(k, device="meta"))

    @staticmethod
    def zeros(*a, **k):
        return torch.empty(*a, **dict(k, device="meta"))

    @staticmethod
    def empty_like(t, **k):
        return torch.empty_like(t, **dict(k, device="meta"))


@contextlib.contextmanager
def _patched(obj, **attrs):
    old = {k: getattr(obj, k) for k in attrs}
    for k, v in attrs.items():
        setattr(obj, k, v)
    try:
        yield
    finally:
        for k, v in old.items():
            setattr(obj, k, v)


def _meta(*shape):
    return torch.empty(shape, dtype=torch.bfloat16, device="meta")


def record(cfg):
    """{"fwd": [...], "bwd": [...]}: the calls of one configuration, through the drivers of the imported package."""
    from burst_attn import burst_attn_interface as bai, chunk_ops, flash_triton, host_stream
    log = []
    ops = RecordingOps(log)
    chunk_ops._set_ops_for_testing(ops)
    env = os.environ.get("BA_L2_BLOCK")
    os.environ["BA_L2_BLOCK"] = str(cfg.get("blk", 32768))
    planner = "band" in inspect.signature(bai._ring_forward).parameters  # else the commit with the mask-free planner
    try:
        causal, window = cfg["causal"], cfg.get("window", (-1, -1))
        plan = {}
        if cfg["kind"] == "ring":
            B, S, H, D, layout = 1, cfg["S"], cfg.get("H", 2), cfg.get("D", 16), cfg["layout"]
            topo = _Topology(cfg["W"], cfg["rank"], log)
            q, k, v = _meta(B, S, H, D), _meta(B, S, H, D), _meta(B, S, H, D)
            alibi = torch.empty((B, H), dtype=torch.float32, device="meta") if cfg.get("alibi") else None
            band = bai._check_window(window, causal)
            if planner:
                fwd = (layout, band, topo, alibi)
                bwd = (layout, band, topo, False, alibi)
            else:
                mode = "none" if not causal else layout
                fwd = (mode, topo, band, layout, alibi)
                bwd = (mode, topo, False, band, layout, alibi)
            out, lse = bai._ring_forward(q, k, v, 0.125, 1, *fwd)
            plan["fwd"], log[:] = list(log), []
            bai._ring_backward(_meta(B, S, H, D), q, k, v, out, lse, 0.125, 1, *bwd)
        elif cfg["kind"] == "local":
            B, H, D = 1, 2, 16
            q, k, v = (_meta(B, n, H, D).requires_grad_() for n in (cfg["Sq"], cfg["Sk"], cfg["Sk"]))
            slopes = torch.empty((H,), dtype=torch.float32, device="meta") if cfg.get("alibi") else None
            with _patched(flash_triton, _check_alibi=lambda s, q, d: None if s is None else s.expand(B, H)):
                o = flash_triton.flash_attn_func(q, k, v, None, causal, None, window, slopes)
                plan["fwd"], log[:] = list(log), []
                torch.autograd.grad(o, (q, k, v), _meta(*o.shape))
        else:
            B, S, H, D, blk = 1, cfg["S"], 2, 16, cfg["blk"]
            q, k, v = _meta(B, S, H, D), _meta(B, S, H, D), _meta(B, S, H, D)
            how = bai._check_window(None, causal) if planner else causal
            with _patched(host_stream, torch=_MetaTorch()), \
                    _patched(torch.Tensor, is_pinned=lambda t: True, record_stream=lambda t, s: None):
                _, saved = host_stream.forward(q, k, v, 0.125, 1, how, blk)
                plan["fwd"], log[:] = list(log), []
                host_stream.backward(_meta(B, S, H, D), saved, 0.125, 1, how, blk, False)
        plan["bwd"] = list(log)
        return plan
    finally:
        chunk_ops._set_ops_for_testing(None)
        if env is None:
            os.environ.pop("BA_L2_BLOCK", None)
        else:
            os.environ["BA_L2_BLOCK"] = env


def _launch(e):
    """(kind, rows, keys, band normalised by ``_band``, ALiBi distance) of a recorded attention launch."""
    from burst_attn.burst_attn_interface import _band
    (q0, qn), (k0, kn) = e[1], e[2]
    return [e[0], q0, qn, k0, kn, *_band(qn, kn, e[5], e[4] if e[3] else None), e[-1]]


def _cover(log):
    """Per ring round and row the keys attended, as joined intervals [first, last, ALiBi distance of row 0 to key 0
    of the round]; a key attended twice by one row in one round fails."""
    out, cur = [], {}
    for e in log + [["wait"]]:
        if e[0] == "wait":
            out.append(sorted((a, _join(iv)) for a, iv in cur.items()))
            cur = {}
        elif e[0] in ("fwd", "bwd"):
            _, q0, qn, k0, kn, lo, hi, alibi = _launch(e)
            inv = None if alibi is None else alibi[0] - alibi[1] * (q0 - k0)
            for a in range(qn):
                c0, c1 = 0 if lo is None else max(0, a + lo), kn - 1 if hi is None else min(kn - 1, a + hi)
                if c0 <= c1:
                    cur.setdefault(q0 + a, []).append((k0 + c0, k0 + c1, inv))
    return out


def _join(iv):
    iv = sorted(iv)
    out = [list(iv[0])]
    for c0, c1, inv in iv[1:]:
        assert c0 > out[-1][1], f"key {c0} attended twice"
        if c0 == out[-1][1] + 1 and inv == out[-1][2]:
            out[-1][1] = c1
        else:
            out.append([c0, c1, inv])
    return out


def _digest(x):
    return hashlib.sha1(json.dumps(x).encode()).hexdigest()[:12]


def summary(cfg, plan):
    """What the fixture keeps of a plan.  Without window or ALiBi: [digest of the forward's launches and round ends,
    digest of the backward's launches, round ends and casts, rows the forward casts].  With one: [digest of the keys
    each row attends per round, forward and backward, number of forward launches, of backward launches]."""
    att = lambda d, kinds: [_launch(e) if e[0] in ("fwd", "bwd") else e for e in plan[d] if e[0] in kinds]  # noqa: E731
    if plain(cfg):
        return [_digest(att("fwd", ("fwd", "wait"))), _digest(att("bwd", ("bwd", "wait", "cast"))),
                sum(e[1][1] for e in plan["fwd"] if e[0] == "cast")]
    return [_digest([_cover(plan["fwd"]), _cover(plan["bwd"])]),
            sum(e[0] == "fwd" for e in plan["fwd"]), sum(e[0] == "bwd" for e in plan["bwd"])]


def main():
    pkg = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "burst-attention_b200")
    dest = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "plans.json")
    sys.path.insert(0, os.path.abspath(pkg))
    with open(dest, "w") as f:
        f.write("{\n" + ",\n".join(f"{json.dumps(key(c))}: {json.dumps(summary(c, record(c)))}" for c in CONFIGS)
                + "\n}\n")
    print(f"{len(CONFIGS)} configurations -> {dest}")


if __name__ == "__main__":
    main()
