#!/usr/bin/env python
"""Install the original ShallowSpeed (siboehm/ShallowSpeed, pure Python) into oracle/_ref/ for the benchmark's
reference arm (`bench.py --impl reference`, baseline/run_reference.py) and for regenerating tests/golden/.

The original is not part of this repository.  Its checkout is taken from $SSB_REFERENCE_SRC, else from the default
location below; when neither exists nothing is installed and the reference arm reports itself unavailable.
Installing = copying its `shallowspeed` package (it has no native code and no dependencies beyond NumPy).

    python oracle/build_reference.py [SRC]
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_SRC = "/root/reference"          # where a checkout of the original is conventionally mounted


def source_dir(src=None):
    src = src or os.environ.get("SSB_REFERENCE_SRC") or DEFAULT_SRC
    return src if os.path.isfile(os.path.join(src, "shallowspeed", "pipe.py")) else None


def installed():
    return os.path.isfile(os.path.join(REF_DIR, "shallowspeed", "pipe.py"))


def install(src=None):
    """Copy the original's package into oracle/_ref/shallowspeed (replacing an older copy).  Returns the install
    directory, or None when no checkout of the original is available."""
    src = source_dir(src)
    if src is None:
        return None
    dst = os.path.join(REF_DIR, "shallowspeed")
    tmp = dst + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(os.path.join(src, "shallowspeed"), tmp, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return REF_DIR


if __name__ == "__main__":
    where = install(sys.argv[1] if len(sys.argv) > 1 else None)
    print(f"reference installed in {where}" if where else "no checkout of the original ShallowSpeed found; nothing installed")
