"""Import the unmodified reference package from baseline/_ref/.

pykg2vec imports hyperopt (common.py:8-9), seaborn and matplotlib (utils/visualization.py:7-15) at
module scope; none of them is installed in this image and none is on the scored path, so empty stub
modules are registered first (SURVEY.md Appendix A).  Nothing of the reference is modified."""
import os
import sys
import types

REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def available(ref_dir=REF_DIR):
    return os.path.isdir(os.path.join(ref_dir, "pykg2vec"))


def install_stubs():
    if "hyperopt" not in sys.modules:
        ho = types.ModuleType("hyperopt")
        ho.hp = types.SimpleNamespace()
        for n in ("fmin", "tpe", "Trials", "STATUS_OK", "space_eval"):
            setattr(ho, n, None)
        pyll = types.ModuleType("hyperopt.pyll")
        base = types.ModuleType("hyperopt.pyll.base")
        base.scope = types.SimpleNamespace()
        sys.modules.update({"hyperopt": ho, "hyperopt.pyll": pyll, "hyperopt.pyll.base": base})
    if "seaborn" not in sys.modules:
        sb = types.ModuleType("seaborn")
        sb.set_style = lambda *a, **k: None
        sys.modules["seaborn"] = sb
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.colors = types.SimpleNamespace()
        mpl.pyplot = plt
        sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": plt})


def load(ref_dir=REF_DIR):
    """-> the imported `pykg2vec` package installed in ref_dir (default baseline/_ref; raises ImportError when
    it is not installed there)."""
    if not available(ref_dir):
        raise ImportError("%s/pykg2vec not found" % ref_dir)
    install_stubs()
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    import pykg2vec
    return pykg2vec
