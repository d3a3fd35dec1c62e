#!/usr/bin/env python
"""Recipe for oracle/_ref/: a verbatim, UNMODIFIED copy of the reference's Python package for use as the CPU baseline and as the
checker of the drop-in claim.

TEST / BENCH INFRASTRUCTURE ONLY (see oracle/__init__.py).  The reference (RookieJunChen/FullSubNet-plus) is pure Python; it
"builds" by being copied from its checkout: FSN_REFERENCE_SRC, by default /root/reference.  oracle/_ref/ is listed in .gitignore
(reference sources never enter the history).  Outputs go ONLY into oracle/_ref/.

    python oracle/make_ref.py            # no-op (keeps a previous copy) when the checkout is absent
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("FSN_REFERENCE_SRC") or "/root/reference"
DST = os.path.join(HERE, "_ref")
# the inference path only: models, acoustics, inferencers, the inference dataset, the loader utilities and the shipped config
KEEP_DIRS = ("speech_enhance", "config")


def make(force=False):
    if not os.path.isdir(SRC):
        return os.path.isdir(os.path.join(DST, "speech_enhance"))
    stamp = os.path.join(DST, ".copied")
    if os.path.exists(stamp) and not force:
        return True
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    os.makedirs(DST)
    for d in KEEP_DIRS:
        shutil.copytree(os.path.join(SRC, d), os.path.join(DST, d),
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "*.wav", "*.tar", "*.pth"))
    shutil.copy(os.path.join(SRC, "LICENSE"), os.path.join(DST, "LICENSE"))
    with open(stamp, "w") as f:
        f.write("verbatim copy of the reference's speech_enhance/ and config/ made by oracle/make_ref.py\n")
    return True


if __name__ == "__main__":
    ok = make(force="--force" in sys.argv)
    print("oracle/_ref:", "ready" if ok else f"unavailable (no reference checkout at {SRC} and no previous copy)")
