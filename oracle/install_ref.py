"""TEST INFRASTRUCTURE: copy the UNMODIFIED reference (facebookresearch/SlowFast) into the git-ignored oracle/_ref/.

``__graft_entry__.build()`` runs this.  The comparison tests, the driver tests and bench.py's reference arm import the
reference from there through oracle/refshim.py, so they run wherever the built tree goes, including machines without a
reference checkout.  Source: $SLOWFAST_REFERENCE_SRC, else /root/reference.  When no readable source exists the step
does nothing, and an oracle/_ref/ built earlier is kept.

What is copied is what the reference's own ``pip install`` ships (the pure-Python ``slowfast`` package) plus the plain
files of the checkout the tools read: the driver scripts (tools/), the yaml configs and ava_evaluation/.  Nothing is
edited; every .py file is checked byte for byte against the source.
"""
from __future__ import annotations

import hashlib
import os
import shutil
from pathlib import Path

DST = Path(__file__).resolve().parent / "_ref"
PARTS = ("slowfast", "tools", "configs", "ava_evaluation")


def _source() -> Path | None:
    for cand in (os.environ.get("SLOWFAST_REFERENCE_SRC"), "/root/reference"):
        if not cand:
            continue
        p = Path(cand)
        try:
            if (p / "slowfast").is_dir() and (p / "configs").is_dir() and os.access(p / "slowfast", os.R_OK | os.X_OK):
                return p
        except OSError:
            continue
    return None


def _py_digest(root: Path) -> str:
    h = hashlib.sha256()
    for f in sorted(root.rglob("*.py")):
        if "__pycache__" in f.parts:
            continue
        rel = f.relative_to(root).as_posix()
        if rel.split("/")[0] not in ("slowfast", "tools"):
            continue
        h.update(rel.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def install(verbose: bool = False) -> Path | None:
    """Copy the reference into oracle/_ref/ (skipped when it is already there and identical).  Returns the tree, or None
    when there is neither a source nor an earlier copy."""
    src = _source()
    if src is None:
        return DST if (DST / "slowfast").is_dir() else None
    want = _py_digest(src)
    stamp = DST / ".digest"
    if stamp.is_file() and stamp.read_text().strip() == want:
        return DST
    tmp = DST.with_name("_ref.tmp")
    shutil.rmtree(tmp, ignore_errors=True)
    tmp.mkdir(parents=True)
    for part in PARTS:
        if (src / part).is_dir():
            shutil.copytree(src / part, tmp / part, ignore=shutil.ignore_patterns("__pycache__"))
    got = _py_digest(tmp)
    if got != want:
        shutil.rmtree(tmp, ignore_errors=True)
        raise RuntimeError(f"copy of the reference at {src} is not byte-identical")
    (tmp / ".digest").write_text(want + "\n")
    shutil.rmtree(DST, ignore_errors=True)
    tmp.rename(DST)
    if verbose:
        print(f"reference installed: {DST}")
    return DST


if __name__ == "__main__":
    print(install(verbose=True))
