#!/usr/bin/env python
"""Recipe for oracle/_ref/: an UNMODIFIED copy of the reference tree (ActiveVisionLab/nope-nerf, pure Python, 540 KB).

    python oracle/vendor_ref.py           # $NOPE_NERF_REFERENCE (default: ../reference beside this repository) -> oracle/_ref

The reference is Python, so "building" it is a verbatim copy; build() runs this recipe where a readable reference checkout
exists and does nothing elsewhere.  oracle/_ref/ is listed in .gitignore (reference sources never enter this repository's
history).  Consumers (test infrastructure only, never the product path): oracle/ref_harness.py -> bench.py --impl reference,
bench.py's `reference_cuda` record, the generators of the stored reference results (tools/make_golden*.py),
tools/psnr_parity.py and the train.py plumbing test.  A MANIFEST (sha256 per file) is written so a consumer can prove the copy
is unmodified.
"""
import hashlib
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get("NOPE_NERF_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference"))
DST = os.path.join(ROOT, "oracle", "_ref")
SKIP_DIRS = {".git", "__pycache__"}


def _files(base):
    for d, dirs, files in os.walk(base):
        dirs[:] = sorted(x for x in dirs if x not in SKIP_DIRS)
        for f in sorted(files):
            if f.endswith(".pyc") or f == "MANIFEST.sha256":
                continue
            yield os.path.relpath(os.path.join(d, f), base)


def _sha(p):
    h = hashlib.sha256()
    with open(p, "rb") as f:
        h.update(f.read())
    return h.hexdigest()


def vendor(force=False):
    """returns True when oracle/_ref is present (copied now or earlier)"""
    if not os.path.isdir(SRC) or not os.access(SRC, os.R_OK | os.X_OK):
        return os.path.isdir(DST)
    if os.path.isdir(DST) and not force:
        man = os.path.join(DST, "MANIFEST.sha256")
        if os.path.exists(man):
            want = dict(l.strip().split("  ", 1)[::-1] for l in open(man) if l.strip())
            if all(os.path.exists(os.path.join(DST, f)) and _sha(os.path.join(DST, f)) == h for f, h in want.items()) and \
                    set(want) == set(_files(SRC)):
                return True
        shutil.rmtree(DST)
    os.makedirs(DST, exist_ok=True)
    lines = []
    for rel in _files(SRC):
        dst = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, rel), dst)
        lines.append("%s  %s" % (_sha(dst), rel))
    with open(os.path.join(DST, "MANIFEST.sha256"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return True


if __name__ == "__main__":
    ok = vendor(force="--force" in sys.argv)
    print("oracle/_ref:", "ready" if ok else "unavailable (no %s here)" % SRC)
