"""The unmodified reference package (build()'s copy in the git-ignored oracle/_ref/minisgl_site, see
oracle/reference_site.py) imported into the test process for the duration of one test.

The product package decides at import time whether it runs inside mini-sglang (attention/base.py), so the
reference must not stay importable for the tests that follow: the fixture takes it off ``sys.path`` and out
of ``sys.modules`` again.  Tests that use it skip when build() found no reference checkout."""
from __future__ import annotations

import sys
from pathlib import Path

import pytest

SITE = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "minisgl_site"


def _drop_reference_modules() -> None:
    for name in [m for m in sys.modules if m == "minisgl" or m.startswith("minisgl.")]:
        del sys.modules[name]


@pytest.fixture
def minisgl_ref(b200):
    """The reference's ``minisgl`` package, importable inside the test; requests ``b200`` first so the product
    package is already imported stand-alone."""
    if not (SITE / "minisgl" / "core.py").is_file():
        pytest.skip("reference package not installed (build() copies it when a reference checkout is readable)")
    sys.path.insert(0, str(SITE))
    try:
        import minisgl.attention.base
        import minisgl.layers.attention

        yield sys.modules["minisgl"]
    finally:
        sys.path.remove(str(SITE))
        _drop_reference_modules()
