#!/usr/bin/env python
"""Stages the UNMODIFIED upstream PaSCo sources under oracle/_ref/ (git-ignored, never committed) for the drop-in tests.

    PASCO_REFERENCE=<upstream PaSCo checkout> python oracle/stage_reference.py

Without PASCO_REFERENCE the checkout is looked for at /root/reference, then in a directory named `reference` next to
this repository.  Its setup.py uses
find_packages() but `pasco/` has no __init__.py, so installing it yields an empty wheel; what the project's documented
editable install gives a user is the source tree on sys.path, so `pasco/` and `scripts/` are copied verbatim.  The
product never imports oracle/_ref (only tests/test_dropin_reference.py does).
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def source() -> str:
    if os.environ.get("PASCO_REFERENCE"):
        return os.environ["PASCO_REFERENCE"]
    candidates = ("/root/reference", os.path.join(os.path.dirname(ROOT), "reference"))
    return next((c for c in candidates if os.path.isdir(os.path.join(c, "pasco"))), candidates[0])


def staged() -> bool:
    return os.path.isdir(os.path.join(DST, "pasco"))


def stage() -> bool:
    """Copies pasco/ and scripts/ of the upstream checkout into oracle/_ref; False if there is no checkout."""
    src = source()
    if not os.path.isdir(os.path.join(src, "pasco")):
        return False
    for d in ("pasco", "scripts"):
        shutil.rmtree(os.path.join(DST, d), ignore_errors=True)
        shutil.copytree(os.path.join(src, d), os.path.join(DST, d), ignore=shutil.ignore_patterns("__pycache__", "*.pth"))
    return True


if __name__ == "__main__":
    print(f"staged {source()} under {DST}" if stage() else f"no upstream checkout at {source()}: nothing staged")
