"""Recipe for ``oracle/_ref/``: what bench.py's reference-on-this-GPU arm (``tools/reference_gpu.py``) runs.

The reference project is pure Python, so there is nothing to compile: its ``nisqa`` package is copied as it lies
(a namespace package, nothing added or edited) to ``oracle/_ref/nisqa``.  ``oracle/_ref/`` is git-ignored and is not
part of this repository.  The reference checkout is ``$NISQA_REFERENCE_DIR``, by default ``/root/reference`` (the
location SURVEY.md was written against); without it the recipe does nothing and the arm reports itself unavailable.

    python -m oracle.build_ref
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
REFERENCE_DIR = os.environ.get("NISQA_REFERENCE_DIR", "/root/reference")


def reference_dir():
    """The reference checkout, for the tools that read it directly (the golden generators); exits with a clear
    message when it is absent."""
    if not os.path.isfile(os.path.join(REFERENCE_DIR, "nisqa", "NISQA_model.py")):
        raise SystemExit("no reference checkout at %r: set NISQA_REFERENCE_DIR to the reference project's directory"
                         % REFERENCE_DIR)
    return REFERENCE_DIR


def build():
    """Copy the reference package to oracle/_ref/nisqa; returns False (and changes nothing) without a checkout."""
    pkg = os.path.join(REFERENCE_DIR, "nisqa")
    if not os.path.isfile(os.path.join(pkg, "NISQA_model.py")):
        return False
    dst = os.path.join(REF_OUT, "nisqa")
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    os.makedirs(REF_OUT, exist_ok=True)
    shutil.copytree(pkg, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return True


if __name__ == "__main__":
    print(build())
