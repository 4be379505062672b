"""Two ways to make the reference's import paths resolve to the H100-native modules.

1. Path overlay: put THIS directory ahead of the reference checkout on ``sys.path``.  The overlay
   packages under ``sudo_rm_rf/`` hold only the accelerated modules and extend their ``__path__``
   with the reference's same-named directories, so everything else (``dnn.losses``, the argument
   parsers, ``dnn.utils``, the other model families) is still the reference's own code.
2. ``install()``: leave ``sys.path`` alone (reference checkout importable as usual) and register a
   meta-path finder that redirects exactly the accelerated module names.

Reference call sites this serves: README.md:70-72, dnn/experiments/run_improved_sudormrf.py:23-29,
utils/simple_whamr_evaluation.py:40-44.
"""
import importlib.abc
import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))

#: reference module name -> overlay file (relative to this directory)
REDIRECTS = {
    "sudo_rm_rf.dnn.models.improved_sudormrf": "sudo_rm_rf/dnn/models/improved_sudormrf.py",
    "sudo_rm_rf.dnn.models.groupcomm_sudormrf_v2": "sudo_rm_rf/dnn/models/groupcomm_sudormrf_v2.py",
    "sudo_rm_rf.dnn.models.causal_improved_sudormrf_v3": "sudo_rm_rf/dnn/models/causal_improved_sudormrf_v3.py",
    "sudo_rm_rf.dnn.models.sudormrf": "sudo_rm_rf/dnn/models/sudormrf.py",
    "sudo_rm_rf.dnn.experiments.utils.mixture_consistency":
        "sudo_rm_rf/dnn/experiments/utils/mixture_consistency.py",
}


class _Redirect(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
        rel = REDIRECTS.get(fullname)
        if rel is None:
            return None
        return importlib.util.spec_from_file_location(fullname, os.path.join(_HERE, rel))


_finder = _Redirect()


def install():
    """Redirect the accelerated module names (idempotent).  Call before the reference's imports."""
    if _finder not in sys.meta_path:
        sys.meta_path.insert(0, _finder)
    for name in REDIRECTS:           # drop already-imported reference versions
        mod = sys.modules.get(name)
        if mod is not None and not (getattr(mod, "__file__", "") or "").startswith(_HERE):
            del sys.modules[name]


def uninstall():
    if _finder in sys.meta_path:
        sys.meta_path.remove(_finder)
