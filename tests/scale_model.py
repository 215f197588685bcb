"""The fp64 oracle and the 16-bit model of ``lowp_model`` for whole heads of a problem too big for one score matrix.

``run`` takes one whole-sequence call -- Sq rows against Sk keys under one kernel mask (``mask_oracle.mask_of``:
None, ``("causal_offset", off)``, ``("band", lo, hi)`` or ``("doc", lo, hi, cu, q_pos0, k_pos0, pstride)``) and
optional ALiBi ``(slopes [B, H], dist0, pstride)`` -- and cuts it into blocks of rows.  Each row block is one chain of
its own: the keys it can see (``key_range``), cut at the given key ``seams`` into chunks that carry the state from one
to the next, with the whole call's mask and ALiBi restated for each chunk's first row and first key (``restate``).  A
window or a document then costs in proportion to the pairs it lets through.

Per row block the truth is ``lowp_model.oracle_chain`` and the model ``lowp_model.lowp_chain``.  O, lse and dQ are
row-local, so each block gives its rows' final values; dK and dV add up over the blocks, in fp64 for the truth and in
fp32 for the model (the model is a yardstick of the kernels' error, not a bitwise twin, so its fp32 summation order
does not matter).  The comparator's scales come out of the same ``error_sums`` / ``finish_scales`` / ``magnitudes``
``oracle_chain`` uses: per row for O and dQ, per key for dK and dV with the blocks' per-key sums added before they are
finished.  What ``run`` returns is what ``lowp_model.assert_api_within_model`` takes.

Only the listed query heads are computed; they must cover whole K/V groups, so that dK and dV of every K/V head
they read are complete.  Everything runs on the device the inputs live on, with fp32 matmuls at full precision.
"""
from __future__ import annotations

import contextlib

import torch

import lowp_model as lm
import mask_oracle as mo

NEG_INF = float("-inf")


@contextlib.contextmanager
def full_fp32():
    """fp32 matmuls at full precision (no TF32) inside, the previous settings restored after: the fp32 model would
    otherwise round its products to 10 mantissa bits and stop being a model of the kernels' fp32 accumulation."""
    prec = torch.get_float32_matmul_precision()
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.set_float32_matmul_precision("highest")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(prec)
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32


def _first_at(p0, ps, x):
    """The first index i >= 0 with p0 + ps i >= x."""
    return max(0, -((p0 - x) // ps))


def key_range(mask, r0, r1, sk):
    """[k0, k1): the keys rows [r0, r1) of the whole call can see under its ``mask`` (empty when k0 >= k1)."""
    k0, k1 = 0, sk
    if mask is None:
        return k0, k1
    if mask[0] == "causal_offset":
        return k0, max(0, min(sk, r1 + int(mask[1])))
    lo, hi = mask[1], mask[2]
    if lo is not None:
        k0 = max(k0, r0 + int(lo))
    if hi is not None:
        k1 = min(k1, r1 + int(hi))
    if mask[0] == "doc":
        _, _, _, cu, qp, kp, ps = mask
        d0, d1 = (int(mo.doc_ids([qp + ps * r], cu)[0]) for r in (r0, r1 - 1))
        k0 = max(k0, _first_at(kp, ps, cu[d0]))
        if d1 + 1 < len(cu) - 1:  # positions past the last boundary count as the last document (mo.doc_ids)
            k1 = min(k1, _first_at(kp, ps, cu[d1 + 1]))
    return k0, k1


def restate(mask, alibi, r0, k0):
    """The whole call's ``mask`` and ``alibi`` as one chunk whose first row is row r0 and first key key k0."""
    dr = r0 - k0
    if mask is not None:
        if mask[0] == "causal_offset":
            mask = ("causal_offset", int(mask[1]) + dr)
        else:
            lo, hi = (None if x is None else int(x) + dr for x in mask[1:3])
            mask = ("band", lo, hi) if mask[0] == "band" else \
                ("doc", lo, hi, mask[3], mask[4] + mask[6] * r0, mask[5] + mask[6] * k0, mask[6])
    if alibi is not None:
        slopes, dist0, ps = alibi
        alibi = (slopes, int(dist0) + ps * dr, ps)
    return mask, alibi


def _groups(heads, H, Hkv):
    """The listed query heads as whole K/V groups: [(K/V head, [its query heads])]."""
    G = H // Hkv
    heads = sorted(set(int(h) for h in heads))
    groups = []
    for hk in sorted({h // G for h in heads}):
        members = list(range(hk * G, hk * G + G))
        assert all(h in heads for h in members), (
            f"query heads {heads} split K/V head {hk}'s group {members}: its dK and dV would be incomplete")
        groups.append((hk, members))
    return groups


def run(q, k, v, do, scale, mask=None, alibi=None, heads=None, block=2048, seams=(), mutant=None, mutant_rows=None,
        drop_keys=(), truth=True):
    """The truth and the model of heads ``heads`` (default: all) of one whole-sequence call, in row blocks of
    ``block`` rows (see the module docstring).

    q, do [B,Sq,H,D] and k, v [B,Sk,Hkv,D] in 16 bit, on the device to compute on; ``alibi`` slopes by query head.
    ``seams``: key indices where every row block's keys are cut into chunks that carry the state across (the
    kernels' L2 split).  Faults for the comparator's own tests, in the model only: ``mutant`` (one of lowp_model's
    mutant lists) in the row blocks that hold a row of ``mutant_rows`` (a range; default all), and ``drop_keys``, keys
    no row of the model sees (a -inf key bias; not with ALiBi).  ``truth=False`` skips the fp64 oracle.

    Returns dict(heads, kv_heads, model, truth): model dict(o, lse, dq, dk=[dk], dv=[dv]) in the input dtype (o) and
    fp32; truth dict(o, lse, dq, dk=[dk], dv=[dv], rss, e32, mag, absmax) in fp64.  O, dQ: [B,Sq,len(heads),D]; lse and
    absmax: [B,len(heads),Sq]; dK, dV: [B,Sk,len(kv_heads),D]."""
    assert not (drop_keys and alibi is not None), "drop_keys acts through a key bias, which ALiBi chunks do not take"
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    dev = q.device
    groups = _groups(range(H) if heads is None else heads, H, Hkv)
    heads = [h for _, hs in groups for h in hs]
    kv_heads = [hk for hk, _ in groups]
    nh, nkv = len(heads), len(kv_heads)
    f32, f64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.float64, device=dev)
    model = dict(o=torch.zeros(B, Sq, nh, D, dtype=q.dtype, device=dev), lse=torch.full((B, nh, Sq), NEG_INF, **f32),
                 dq=torch.zeros(B, Sq, nh, D, **f32), dk=torch.zeros(B, Sk, nkv, D, **f32),
                 dv=torch.zeros(B, Sk, nkv, D, **f32))
    ref = dict(o=torch.zeros(B, Sq, nh, D, **f64), lse=torch.full((B, nh, Sq), NEG_INF, **f64),
               dq=torch.zeros(B, Sq, nh, D, **f64), dk=torch.zeros(B, Sk, nkv, D, **f64),
               dv=torch.zeros(B, Sk, nkv, D, **f64), absmax=torch.zeros(B, nh, Sq, **f64))
    rows = {n: torch.zeros(B, Sq, nh, **f64) for n in ("o", "dq", "dq_coh", "e32_dq")}  # per row
    keys = {n: torch.zeros(B, Sk, nh, **f64) for n in ("dk", "dk_coh", "dv", "e32_dk")}  # per key and query head
    with full_fp32():
        for gi, (hk, hs) in enumerate(groups):
            h0, h1 = gi * len(hs), (gi + 1) * len(hs)  # this group's query heads among ``heads``
            qg, dog = q[:, :, hs[0]:hs[-1] + 1], do[:, :, hs[0]:hs[-1] + 1]
            kg, vg = k[:, :, hk:hk + 1], v[:, :, hk:hk + 1]
            al = None if alibi is None else (alibi[0][:, hs[0]:hs[-1] + 1], alibi[1], alibi[2])
            for r0 in range(0, Sq, block):
                r1 = min(Sq, r0 + block)
                k0, k1 = key_range(mask, r0, r1, Sk)
                if k1 <= k0:
                    continue  # no row of the block sees a key: O = 0, lse = -inf, no gradient
                cuts = [k0] + [s for s in sorted(seams) if k0 < s < k1] + [k1]
                ks = [kg[:, a:b] for a, b in zip(cuts, cuts[1:])]
                vs = [vg[:, a:b] for a, b in zip(cuts, cuts[1:])]
                chunks = [restate(mask, al, r0, a) for a in cuts[:-1]]
                masks = [m for m, _ in chunks]
                alibis = None if al is None else [a for _, a in chunks]
                qb, dob = qg[:, r0:r1], dog[:, r0:r1]
                biases = None
                if drop_keys:
                    biases = []
                    for a, b in zip(cuts, cuts[1:]):
                        kb = torch.zeros(1, len(hs), b - a, **f32)
                        for j in drop_keys:
                            if a <= j < b:
                                kb[..., j - a] = NEG_INF
                        biases.append(kb)
                live = mutant_rows is None or (r0 < mutant_rows.stop and mutant_rows.start < r1)
                m = lm.lowp_chain(qb, ks, vs, dob, scale, masks, biases, mutant if live else None, alibis)
                model["o"][:, r0:r1, h0:h1] = m["o"]
                model["lse"][:, h0:h1, r0:r1] = m["lse"]
                model["dq"][:, r0:r1, h0:h1] = m["dq"]
                for (a, b), dk, dv in zip(zip(cuts, cuts[1:]), m["dk"], m["dv"]):
                    model["dk"][:, a:b, gi:gi + 1] += dk
                    model["dv"][:, a:b, gi:gi + 1] += dv
                del m
                if not truth:
                    continue
                t = lm.oracle_chain(qb, ks, vs, dob, scale, masks, alibis=alibis, device=dev)
                ref["o"][:, r0:r1, h0:h1] = t["o"]
                ref["lse"][:, h0:h1, r0:r1] = t["lse"]
                ref["dq"][:, r0:r1, h0:h1] = t["dq"]
                s = t["sums"]
                for n in rows:
                    rows[n][:, r0:r1, h0:h1] = s[n]
                for c, (a, b) in enumerate(zip(cuts, cuts[1:])):
                    ref["dk"][:, a:b, gi:gi + 1] += t["dk"][c]
                    ref["dv"][:, a:b, gi:gi + 1] += t["dv"][c]
                    for n in keys:
                        keys[n][:, a:b, h0:h1] += s[n][c]
                del t, s
                fb = None
                if al is not None:  # the bias in the block's frame, -slope (|d| - dref), as lowp_alibi.frame_bias
                    fb = []
                    for (a, b), (_, (sl, d0, ps)) in zip(zip(cuts, cuts[1:]), chunks):
                        x = lm.distances(r1 - r0, b - a, d0, ps, dev).abs() - \
                            lm.alibi_dref(r1 - r0, b - a, d0, ps, dev).view(-1, 1)
                        fb.append(-sl.to(dev).double().view(B, -1, 1, 1) * x.double())
                ref["absmax"][:, h0:h1, r0:r1] = lm.scores_absmax(qb, ks, scale, masks, fb, device=dev)
                del fb
    out = dict(heads=heads, kv_heads=kv_heads, model=dict(model, dk=[model["dk"]], dv=[model["dv"]]))
    if truth:
        kx = lm._kv_heads(k[:, :, kv_heads], nh)
        vx = lm._kv_heads(v[:, :, kv_heads], nh)
        sums = dict(rows, **{n: [keys[n]] for n in keys})
        out["truth"] = dict(ref, dk=[ref["dk"]], dv=[ref["dv"]], mag=lm.magnitudes(q[:, :, heads], [kx], [vx],
                                                                                   do[:, :, heads], scale),
                            **lm.finish_scales(sums, ref["o"], nkv, [Sk]))
    return out


def check_api(name, out, q, k, v, do, mask=None, alibi=None, heads=None, block=2048, seams=()):
    """Heads ``heads`` (whole K/V groups) of one public call's ``out = (o, dq, dk, dv)`` on q, k, v, do (default
    scale) against ``run``'s truth and model: exactly 0 where nothing is visible, and within the model bound
    (``lowp_model.assert_api_within_model``)."""
    o, dq, dk, dv = out
    r = run(q, k, v, do, q.shape[-1] ** -0.5, mask, alibi, heads=heads, block=block, seams=seams)
    hs, kvs = r["heads"], r["kv_heads"]
    got = dict(o=pick(o, hs), dq=pick(dq, hs), dk=pick(dk, kvs), dv=pick(dv, kvs))
    t = r["truth"]
    dead = torch.isinf(t["lse"]).permute(0, 2, 1)  # [B,S,h]: rows that see nothing
    assert int(got["o"][dead].count_nonzero()) == 0 and int(got["dq"][dead].count_nonzero()) == 0, name
    blind = t["rss"]["dv"] == 0  # [B,S,hkv]: keys no row sees
    assert int(got["dk"][blind].count_nonzero()) == 0 and int(got["dv"][blind].count_nonzero()) == 0, name
    lm.assert_api_within_model(name, got, t, r["model"], q.dtype)


def pick(t, heads, dim=2):
    """The listed heads of a kernel output ([B,S,H,D]: dim 2; [B,H,S]: dim 1), in ``run``'s order."""
    return t.index_select(dim, torch.tensor(heads, device=t.device))
