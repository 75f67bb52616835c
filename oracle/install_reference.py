"""Stage the unmodified reference package (GeeeekExplorer/nano-vllm) under oracle/_ref/, git-ignored.

    python oracle/install_reference.py [<checkout of the reference>]

The reference is pure Python, so staging is a copy of its ``nanovllm`` package.  The checkout is the argument, else
NANOVLLM_REFERENCE, else /root/reference (where the build environment keeps it); build() calls install() with no
argument.  Tools that run the reference next to the product import it from oracle/_ref (both packages are called
``nanovllm``, so they run in a subprocess of their own): oracle/make_golden.py, oracle/make_gpu_golden.py,
oracle/ref_cpu_arm.py (bench.py's CPU arm), baseline/run_reference_gpu.py and profiles/host_bookkeeping.py.
tests/test_gpu_reference_forward.py runs INTEGRATION.md's option B with it (and skips where nothing could be staged);
every other test reads what it compares against from tests/golden/.
"""
from __future__ import annotations

import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_SRC = "/root/reference"


def install(src: str | None = None) -> str:
    """Copy <src>/nanovllm to oracle/_ref/nanovllm unless it is there already.  Returns what happened, in words."""
    src = src or os.environ.get("NANOVLLM_REFERENCE") or DEFAULT_SRC
    if os.path.isdir(os.path.join(DST, "nanovllm")):
        return "present"
    if not os.path.isdir(os.path.join(src, "nanovllm")):
        return f"skipped (no readable reference checkout at {src})"
    tmp = DST + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    try:
        shutil.copytree(os.path.join(src, "nanovllm"), os.path.join(tmp, "nanovllm"),
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    except OSError as e:                   # a partly readable checkout: stage nothing rather than half a package
        shutil.rmtree(tmp, ignore_errors=True)
        return f"skipped ({src}: {e})"
    os.replace(tmp, DST)
    return "installed from " + src


if __name__ == "__main__":
    print("oracle/_ref:", install(sys.argv[1] if len(sys.argv) > 1 else None))
