"""Import the UNMODIFIED reference project (TEST INFRASTRUCTURE).

The reference is an upstream checkout: $LANEFIT_REFERENCE_DIR, else ../reference next to this repository.  ``install()``
(called by ``__graft_entry__.build()``) copies its hot-path modules into oracle/_ref/ (git-ignored), which is used when
the checkout itself is not reachable.  No test and neither ``smoke()`` nor ``bench.py``'s timed path needs it;
``bench.py`` uses it for the reference arm / cpu_baseline only (kind "reference"; without it, the oracle port is timed).
Recipe = SURVEY.md Appendix A: the reference modules use top-level
``import Networks`` and need ``matplotlib`` at import time
(Backprojection_Loss/Networks/utils.py:17-21), which this image lacks -> stub it.
"""
import os
import sys
import types

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE_ROOT = os.environ.get("LANEFIT_REFERENCE_DIR") or os.path.join(os.path.dirname(_REPO), "reference")
INSTALLED_ROOT = os.path.join(_REPO, "oracle", "_ref")
_CANDIDATES = [SOURCE_ROOT, INSTALLED_ROOT]
_HOT_PATH_FILES = ["Networks/__init__.py", "Networks/ERFNet.py", "Networks/LSQ_layer.py", "Networks/gels.py",
                   "Networks/utils.py", "Loss_crit.py"]


def _root():
    for r in _CANDIDATES:
        if os.path.isdir(os.path.join(r, "Backprojection_Loss", "Networks")):
            return r
    return None


REFERENCE_ROOT = _root() or SOURCE_ROOT


def available():
    return _root() is not None


def install(src=SOURCE_ROOT, dst=INSTALLED_ROOT):
    """Copy the reference's hot-path modules (both variants) verbatim from `src` to oracle/_ref.  No-op (False) when
    `src` is absent or unreadable."""
    import shutil
    if not os.access(os.path.join(src, "Backprojection_Loss", "Networks"), os.R_OK | os.X_OK):
        return False
    for variant in ("Backprojection_Loss", "Birds_Eye_View_Loss"):
        for rel in _HOT_PATH_FILES:
            s = os.path.join(src, variant, rel)
            if os.path.exists(s):
                d = os.path.join(dst, variant, rel)
                os.makedirs(os.path.dirname(d), exist_ok=True)
                shutil.copyfile(s, d)
    for extra in ("LICENSE.txt",):
        if os.path.exists(os.path.join(src, extra)):
            shutil.copyfile(os.path.join(src, extra), os.path.join(dst, extra))
    return True


def _stub_matplotlib():
    if "matplotlib" in sys.modules:
        return
    try:
        import matplotlib  # noqa: F401
        return
    except Exception:
        pass
    m = types.ModuleType("matplotlib")
    m.use = lambda *a, **k: None
    p = types.ModuleType("matplotlib.pyplot")
    p.rcParams = {}
    m.pyplot = p
    sys.modules["matplotlib"] = m
    sys.modules["matplotlib.pyplot"] = p


def purge():
    for k in list(sys.modules):
        if k == "Networks" or k.startswith("Networks.") or k in ("Loss_crit",):
            del sys.modules[k]
    sys.path[:] = [p for p in sys.path if not any(p.startswith(r) for r in _CANDIDATES)]


def import_reference(variant="Backprojection_Loss"):
    """Returns a namespace with the reference's Net, define_args, define_init_weights,
    backprojection_loss / Area_Loss, get_homography, Weighted_least_squares,
    ProjectiveGridGenerator, GELS for the given variant directory."""
    root = _root()
    if root is None:
        raise RuntimeError("reference not present at any of " + ", ".join(_CANDIDATES))
    _stub_matplotlib()
    purge()
    sys.path.insert(0, os.path.join(root, variant))
    ns = types.SimpleNamespace()
    import Networks  # noqa: F401
    from Networks import LSQ_layer, ERFNet, utils
    import Loss_crit
    ns.Networks = Networks
    ns.LSQ_layer = LSQ_layer
    ns.ERFNet = ERFNet
    ns.utils = utils
    ns.Loss_crit = Loss_crit
    if variant == "Backprojection_Loss":
        from Networks import gels
        ns.gels = gels
    return ns


def make_args(ns, extra=(), no_cuda=True):
    """argparse Namespace the reference's ``Net(args)`` consumes (utils.py:24-99)."""
    argv = ["--image_dir", "x", "--gt_dir", "y"] + (["--no_cuda"] if no_cuda else []) + list(extra)
    return ns.utils.define_args().parse_args(argv)
