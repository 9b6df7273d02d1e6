"""Stage an unmodified copy of the reference project's Python package and its bundled cinderella sample under
oracle/_ref (git-ignored).  build() runs this where the reference checkout exists; the copy then travels with the
working tree, so the end-to-end tests (tests/test_e2e_cinderella.py) and bench.py's CPU baseline can run the
reference's own ComoRAG code on machines that have no checkout of it.

The checkout is $COMORAG_REFERENCE, else the reference's default location.  The copy is refreshed only when its
recorded checksums no longer describe the checkout.
"""
from __future__ import annotations

import hashlib
import os
import shutil
from typing import Optional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_SRC = "/root/reference"
PARTS = ("src", os.path.join("dataset", "cinderella"))


def _files(base: str):
    for part in PARTS:
        for d, dirs, files in os.walk(os.path.join(base, part)):
            dirs[:] = sorted(x for x in dirs if x != "__pycache__")
            for f in sorted(files):
                if not f.endswith(".pyc"):
                    yield os.path.relpath(os.path.join(d, f), base)


def _sums(base: str) -> str:
    lines = []
    for rel in _files(base):
        with open(os.path.join(base, rel), "rb") as fh:
            lines.append(f"{hashlib.sha256(fh.read()).hexdigest()}  {rel}")
    return "\n".join(lines) + "\n"


def stage(src: Optional[str] = None) -> str:
    """Returns a one-line account of what was done."""
    src = src or os.environ.get("COMORAG_REFERENCE") or DEFAULT_SRC
    if not os.path.isdir(os.path.join(src, "src", "comorag")):
        state = "present" if os.path.isdir(os.path.join(DST, "src", "comorag")) else "absent"
        return f"no reference checkout here; oracle/_ref is {state}"
    want = _sums(src)
    sums = os.path.join(DST, "SHA256SUMS")
    if os.path.isfile(sums) and open(sums).read() == want:
        return "oracle/_ref: staged copy matches the reference checkout"
    shutil.rmtree(DST, ignore_errors=True)
    for rel in _files(src):
        os.makedirs(os.path.dirname(os.path.join(DST, rel)), exist_ok=True)
        shutil.copyfile(os.path.join(src, rel), os.path.join(DST, rel))
    if os.path.isfile(os.path.join(src, "LICENSE")):
        shutil.copyfile(os.path.join(src, "LICENSE"), os.path.join(DST, "LICENSE"))
    with open(sums, "w") as fh:
        fh.write(want)
    return f"oracle/_ref: staged {len(want.splitlines())} files of the reference checkout"


if __name__ == "__main__":
    print(stage())
