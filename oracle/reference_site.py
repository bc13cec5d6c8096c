"""Recipe: place the unmodified reference package (sgl-project/mini-sglang, ``python/minisgl``) into the
git-ignored ``oracle/_ref/minisgl_site`` so that the in-situ harness (tools/insitu.py,
tests/test_gpu_insitu.py) can drive the reference's own LLM -> Scheduler -> Engine stack.

The reference is pure Python (its CUDA parts are JIT-compiled at run time), so "building" it is a copy
of its package tree; nothing of it enters the repository.  The checkout is looked up in
``$MINISGL_REFERENCE`` (the reference's repository root), then at ``/root/reference``.  Without a
readable checkout an existing copy is left as it is; with none at all the in-situ test skips.
"""

from __future__ import annotations

import os
import shutil
from pathlib import Path
from typing import Optional

ROOT = Path(__file__).resolve().parent.parent
SITE = ROOT / "oracle" / "_ref" / "minisgl_site"
DEFAULT_CHECKOUT = Path("/root/reference")


def find_checkout() -> Optional[Path]:
    for cand in (os.environ.get("MINISGL_REFERENCE"), DEFAULT_CHECKOUT):
        if not cand:
            continue
        pkg = Path(cand) / "python" / "minisgl"
        try:
            if (pkg / "core.py").is_file() and os.access(pkg, os.R_OK | os.X_OK):
                return pkg
        except OSError:
            continue
    return None


def installed() -> bool:
    return (SITE / "minisgl" / "core.py").is_file()


def install() -> Optional[Path]:
    """Copy the reference package into SITE (replacing an older copy).  Returns SITE when a copy is in
    place afterwards, None otherwise (no readable checkout and no earlier copy, or a read-only tree)."""
    pkg = find_checkout()
    if pkg is None:
        return SITE if installed() else None
    dest = SITE / "minisgl"
    tmp = SITE / "minisgl.tmp"
    try:
        SITE.mkdir(parents=True, exist_ok=True)
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(pkg, tmp, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        shutil.rmtree(dest, ignore_errors=True)
        tmp.rename(dest)
    except OSError:
        shutil.rmtree(tmp, ignore_errors=True)
    return SITE if installed() else None


if __name__ == "__main__":
    print(install() or "no readable reference checkout found (set MINISGL_REFERENCE)")
