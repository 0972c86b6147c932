"""The unmodified reference package (Sujit-O/pykg2vec @ 492807b) under oracle/_ref/, for the tests that drive
the reference's own Importer / Trainer / Evaluator with this package's classes.

The reference is pure Python, so installing it is a copy of its package directory (what `pip install --target`
places there; its own test suite is left out).  Nothing of it is modified.  The checkout is found at
$PYKG2VEC_REFERENCE, by default /root/reference.  Without it nothing is installed, and the tests that need it
skip."""
import os
import shutil

REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def install(src=None):
    """Copy <src>/pykg2vec to oracle/_ref/pykg2vec.  Returns REF_DIR, or None when there is no reference."""
    src = src or os.environ.get("PYKG2VEC_REFERENCE", "/root/reference")
    pkg = os.path.join(src, "pykg2vec")
    if not os.path.isfile(os.path.join(pkg, "__init__.py")):
        return None
    tmp = os.path.join(REF_DIR, "pykg2vec.tmp")
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(pkg, tmp, ignore=shutil.ignore_patterns("test", "__pycache__", "*.pyc"))
    dst = os.path.join(REF_DIR, "pykg2vec")
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return REF_DIR
