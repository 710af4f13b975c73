"""Drop-in surface of trajnetbaselines.lstm (reference: trajnetbaselines/lstm/__init__.py)."""
from .loss import PredictionLoss, L2Loss
from .lstm import LSTM, LSTMPredictor, drop_distant
from .training import differentiable_rollout
from .shapley import Shapley, shapley, shapley_scenes
from .gridbased_pooling import GridBasedPooling
from .non_gridbased_pooling import HiddenStateMLPPooling, NearestNeighborMLP, AttentionMLPPooling, NearestNeighborLSTM, TrajectronPooling


def __getattr__(name):
    # SampledLSTMPredictor (lstm/sampling.py) builds on multimodal.py, which imports this package: loaded on first use
    if name == 'SampledLSTMPredictor':
        from .sampling import SampledLSTMPredictor
        return SampledLSTMPredictor
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
