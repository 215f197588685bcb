"""Record how the twelve chunk entry points of the C-ABI (``ba_fwd_chunk*`` / ``ba_bwd_chunk*``) reject their
arguments, and keep each call's return code and ``ba_last_error()`` in ``chunk_abi_errors.json``.

The sweep reaches every argument condition of the chunk calls: K/V heads, head dim, empty problem, dtype, mask bits,
scale, grid limits, a reversed band, offsets at the int32 extremes, the ALiBi slopes and position stride, the document
boundaries, counts and positions, and pairs of failing conditions, which pin the order in which each entry point
reports them.  Every call passes null q / k / v / dO, so a call with valid arguments stops at the operand check: no
call reaches a tensor map or a launch, and no GPU is needed.  Pointer arguments that must be non-null (``slopes``,
``cu_seqlens``) are small integers the checks never dereference.

    python tests/golden/make_chunk_abi_errors.py [package dir] [output]

The fixture was recorded from the commit before the chunk calls shared one argument check;
``tests/test_chunk_abi_errors.py`` replays the sweep against the current library."""
import ctypes
import json
import math
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
HEADER = os.path.join(ROOT, "include", "burst_attn_b200.h")

ENTRIES = [f"ba_{d}_chunk{v}" for d in ("fwd", "bwd") for v in ("", "_bias", "_gqa", "_band", "_alibi", "_doc")]
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1

# a valid call of every entry point, by parameter name (each takes those it has); operands are null
BASE = dict(B=1, Sq=128, Sk=128, H=4, H_kv=2, D=128, scale=1.0, mask_mode=1, causal_offset=0, lower_offset=0,
            dtype=1, slopes=16, slopes_stride_b=0, dist0=0, pstride=1, cu_seqlens=16, n_docs=1, q_pos0=0, k_pos0=0)

CASES = [
    {},
    dict(mask_mode=0), dict(mask_mode=2), dict(mask_mode=3, causal_offset=5, lower_offset=-5),
    dict(mask_mode=2, lower_offset=-127), dict(mask_mode=2, lower_offset=-126), dict(mask_mode=2, lower_offset=129),
    # K/V heads
    dict(H_kv=0), dict(H_kv=-2), dict(H_kv=3), dict(H=2, H_kv=4), dict(H=4, H_kv=4), dict(H=4, H_kv=1),
    # head dim
    dict(D=64), dict(D=96), dict(D=0), dict(D=256),
    # empty problem
    dict(B=0), dict(Sq=0), dict(Sk=0), dict(H=0), dict(Sq=-1), dict(B=-3),
    # dtype
    dict(dtype=0), dict(dtype=2), dict(dtype=-1),
    # mask bits
    dict(mask_mode=4), dict(mask_mode=5), dict(mask_mode=7), dict(mask_mode=-1), dict(mask_mode=8),
    # scale
    dict(scale=0.0), dict(scale=-1.0), dict(scale=math.nan), dict(scale=math.inf), dict(scale=-math.inf),
    dict(scale=1e-30),
    # grid limits
    dict(H=65536, H_kv=1), dict(H=65535, H_kv=1), dict(B=65536), dict(B=65535),
    # a reversed band, and offsets at the int32 extremes
    dict(mask_mode=3, causal_offset=0, lower_offset=1), dict(mask_mode=3, causal_offset=-7, lower_offset=-6),
    dict(mask_mode=3, causal_offset=I32_MIN, lower_offset=I32_MIN + 1),
    dict(mask_mode=3, causal_offset=I32_MIN, lower_offset=I32_MIN),
    dict(mask_mode=3, causal_offset=I32_MAX, lower_offset=I32_MAX),
    dict(mask_mode=1, causal_offset=I32_MIN), dict(mask_mode=1, causal_offset=I32_MAX),
    dict(mask_mode=2, lower_offset=I32_MIN), dict(mask_mode=2, lower_offset=I32_MAX),
    # ALiBi slopes and position stride
    dict(slopes=0), dict(slopes=18), dict(slopes=17), dict(slopes_stride_b=-1), dict(slopes_stride_b=-4),
    dict(slopes_stride_b=4), dict(pstride=0), dict(pstride=-1), dict(pstride=8), dict(dist0=-(2 ** 40)),
    # document boundaries, counts and positions
    dict(cu_seqlens=0), dict(cu_seqlens=2), dict(cu_seqlens=6), dict(n_docs=0), dict(n_docs=-1), dict(n_docs=1000),
    dict(q_pos0=-1), dict(k_pos0=-1), dict(q_pos0=-(2 ** 40)), dict(q_pos0=2 ** 31 - 100),
    dict(k_pos0=2 ** 31 - 128), dict(k_pos0=2 ** 31 - 127), dict(q_pos0=2 ** 40), dict(pstride=2 ** 24),
    dict(pstride=2 ** 25),
    # two failing conditions at once: which one each entry point reports first
    dict(mask_mode=4, H_kv=0), dict(mask_mode=4, D=96), dict(mask_mode=6, B=0), dict(mask_mode=2, D=96),
    dict(mask_mode=2, dtype=3), dict(mask_mode=3, H_kv=3), dict(D=96, dtype=3), dict(H_kv=0, D=96),
    dict(B=0, dtype=3), dict(dtype=3, scale=0.0), dict(scale=0.0, B=65536),
    dict(mask_mode=3, lower_offset=1, scale=0.0),
    dict(mask_mode=3, lower_offset=1, H=65536, H_kv=1), dict(mask_mode=3, lower_offset=1, slopes=0),
    dict(mask_mode=3, lower_offset=1, cu_seqlens=0), dict(slopes=0, H_kv=0), dict(slopes=0, mask_mode=4),
    dict(slopes=18, slopes_stride_b=-1), dict(slopes_stride_b=-1, pstride=0), dict(cu_seqlens=0, n_docs=0),
    dict(cu_seqlens=6, pstride=0), dict(n_docs=0, pstride=0), dict(pstride=0, q_pos0=-1),
    dict(q_pos0=-1, k_pos0=2 ** 31), dict(cu_seqlens=0, D=96),
]


def key(case):
    return " ".join(f"{k}={v!r}" for k, v in case.items()) or "valid"


def parameters():
    """{entry point: [parameter names]} of the chunk entry points, from the header."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"\bint\s+(ba_(?:fwd|bwd)_chunk\w*)\s*\(([^)]*)\)\s*;", src):
        out[name] = [p.split()[-1].lstrip("*") for p in params.split(",")]
    assert sorted(out) == sorted(ENTRIES), sorted(out)
    return out


def call(native, L, params, entry, case):
    """[return code, ba_last_error()] of one call of ``entry`` with the arguments of ``case``."""
    vals = dict(BASE, flags=3 if entry.startswith("ba_fwd") else 0, **case)
    args = []
    for p, t in zip(params[entry], getattr(L, entry).argtypes):
        if t is native.ba_tensor4:
            args.append(native.ba_tensor4(None, 0, 0, 0))
        elif t is native.ba_rowstat:
            args.append(native.ba_rowstat(None, 0, 0))
        elif p == "stream":
            args.append(None)
        else:
            args.append(vals[p] or None if t is ctypes.c_void_p else vals[p])
    rc = getattr(L, entry)(*args)
    return [rc, L.ba_last_error().decode()]


def sweep(native):
    """{entry point: {case: [return code, error]}} over every entry point and case."""
    L, params = native.lib(), parameters()
    return {e: {key(c): call(native, L, params, e, c) for c in CASES} for e in ENTRIES}


def main():
    pkg = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "burst-attention_b200")
    dest = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "chunk_abi_errors.json")
    sys.path.insert(0, os.path.abspath(pkg))
    from burst_attn import native
    with open(dest, "w") as f:
        json.dump(sweep(native), f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(ENTRIES)} entry points x {len(CASES)} cases -> {dest}")


if __name__ == "__main__":
    main()
