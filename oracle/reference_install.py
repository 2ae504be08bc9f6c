"""Install the unmodified reference package (lucidrains/vit-pytorch 1.23.6, pure Python) into oracle/_ref/.

A few CPU tests run the reference's own wrapper code (MAE, DistillWrapper, AcceptVideoWrapper, Extractor) on the
drop-in modules. That code cannot be stored in this repository, so build() copies the `vit_pytorch` package out of a
reference checkout into oracle/_ref/ (git-ignored, a build product like the CUDA library). The checkout is taken from
VIT_REFERENCE, else from DEFAULT_CHECKOUT. Without a readable checkout of that version nothing is installed, and
those tests are skipped.

    python -m oracle.reference_install
"""
from __future__ import annotations

import os
import re
import shutil
from pathlib import Path
from typing import Optional

VERSION = "1.23.6"
DEFAULT_CHECKOUT = "/root/reference"
DEST = Path(__file__).resolve().parent / "_ref"


def checkout() -> Optional[Path]:
    """The reference checkout to install from, or None if there is no readable checkout of VERSION."""
    src = Path(os.environ.get("VIT_REFERENCE") or DEFAULT_CHECKOUT)
    try:
        meta = (src / "pyproject.toml").read_text()
        if not (src / "vit_pytorch" / "__init__.py").is_file():
            return None
    except OSError:
        return None
    m = re.search(r'^version\s*=\s*"([^"]+)"', meta, flags=re.M)
    return src if m and m.group(1) == VERSION else None


def install() -> Optional[Path]:
    """Copy <checkout>/vit_pytorch to oracle/_ref/vit_pytorch (replacing an older copy); returns oracle/_ref or None."""
    src = checkout()
    if src is None:
        return None
    tmp = DEST.with_name("_ref.tmp")
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(src / "vit_pytorch", tmp / "vit_pytorch", ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    (tmp / "VERSION").write_text(VERSION + "\n")
    shutil.rmtree(DEST, ignore_errors=True)
    tmp.rename(DEST)
    return DEST


if __name__ == "__main__":
    print(install() or "no reference checkout found: nothing installed")
