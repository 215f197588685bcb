"""Recipe for oracle/_ref: the UNMODIFIED reference (MayDomine/Burst-Attention) made importable next to this
project, for the measurement legs that run the reference itself (baseline/ref_shim.py: bench.py's CPU arm and
tools/ref_on_gpu.py).  The reference's ``burst_attn`` package is pure Python, so "building" it is a copy of that
package into the git-ignored oracle/_ref; nothing of it enters the tracked tree and nothing is edited.

The reference checkout is taken from BA_REFERENCE_DIR (default /root/reference).  Where it does not exist the
recipe does nothing and the measurement legs fall back to the oracle's restatement of the same path.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")


def reference_dir() -> str:
    return os.environ.get("BA_REFERENCE_DIR", "/root/reference")


def build(dst: str = DST) -> bool:
    """Copy <reference>/burst_attn into dst/burst_attn (replacing an older copy).  Returns True when dst holds the
    reference afterwards."""
    src = os.path.join(reference_dir(), "burst_attn")
    if not os.path.isfile(os.path.join(src, "__init__.py")):
        return os.path.isfile(os.path.join(dst, "burst_attn", "__init__.py"))
    tmp = dst + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(src, os.path.join(tmp, "burst_attn"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return True


if __name__ == "__main__":
    ok = build()
    print(f"oracle/_ref: {'reference installed' if ok else 'no reference checkout at ' + reference_dir()}")
    sys.exit(0 if ok else 1)
