"""Import shim for the UNMODIFIED reference.

TEST INFRASTRUCTURE -- never imported by the product package.  The reference's
third-party imports that are absent from this image (SURVEY.md Appendix B) are
replaced by stub modules so `trajnetbaselines.lstm` imports; the tensor-level
calls (LSTM.forward/step, GridBasedPooling.*, PredictionLoss, Trainer.train_batch) never
touch the stubs, except `trajnetplusplustools.Reader.paths_to_xy` / `TrackRow`, which the
reference's LSTMPredictor calls: those two are served by this repo's data helpers.

Where the reference lives:
  * /root/reference          -- the read-only source tree
  * oracle/_ref              -- `oracle/build_ref.py` (run by build()): the same packages compiled to
                                bytecode plus DATA_BLOCK; git-ignored build product, so a machine
                                without the source tree runs the reference tests from it.
`TRAJNET_REFERENCE_ROOT` overrides both.
"""
import os
import sys
import types

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CANDIDATES = [os.environ.get("TRAJNET_REFERENCE_ROOT"), "/root/reference", os.path.join(_REPO, "oracle", "_ref")]


def reference_root():
    for root in _CANDIDATES:
        if root and os.access(os.path.join(root, "trajnetbaselines"), os.R_OK | os.X_OK):
            return root
    return None


REFERENCE_ROOT = reference_root() or "/root/reference"


def reference_available():
    return reference_root() is not None


def _stub(name, **attrs):
    if name in sys.modules:
        mod = sys.modules[name]
        for k, v in attrs.items():
            if not hasattr(mod, k):
                setattr(mod, k, v)
        return mod
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


def import_reference(root=None):
    """Return the reference's `trajnetbaselines` package (stubs registered first)."""
    root = root or reference_root()
    if root is None:
        raise ImportError("reference not present (neither /root/reference nor oracle/_ref)")
    from trajnetplusplusbaselines_b200 import data as _data       # TrackRow / paths_to_xy stand-ins

    class _Reader(object):
        paths_to_xy = staticmethod(_data.paths_to_xy)

    _stub("trajnetplusplustools", Reader=_Reader, TrackRow=_data.TrackRow, SceneRow=_data.SceneRow)
    _stub("trajnetplusplustools.show")
    _stub("trajnetplusplustools.reader", Reader=_Reader)
    _stub("matplotlib")
    _stub("matplotlib.pyplot")
    _stub("matplotlib.font_manager", FontProperties=object)
    _stub("matplotlib.animation")
    _stub("mpl_toolkits")
    _stub("mpl_toolkits.mplot3d")
    _stub("mpl_toolkits.mplot3d.axes3d")
    _stub("pykalman")
    _stub("socialforce")
    _stub("socialforce.potentials", PedPedPotential=object)
    _stub("socialforce.field_of_view", FieldOfView=object)
    _stub("rvo2")
    _stub("pysparkling")
    _stub("pythonjsonlogger")
    if not os.path.isdir(os.path.join(root, "evaluator")):
        _stub("evaluator")
        _stub("evaluator.trajnet_evaluator", trajnet_evaluate=None)
        _stub("evaluator.write_utils", load_test_datasets=None, preprocess_test=_data.preprocess_test, write_predictions=None)
    if root not in sys.path:
        sys.path.insert(0, root)
    import trajnetbaselines  # noqa: E402
    return trajnetbaselines
