"""zaremba_b200: H100-native (sm_90a) implementation of the LSTM-LM hot path of
ahmetumutdurmus/zaremba behind the reference's `model.Model` interface.

    from zaremba_b200 import Model            # drop-in for the reference's model.py
    from zaremba_b200 import Trainer          # fused train / eval step (main.py:109-117, :86-95)
    from zaremba_b200 import sample           # on-device top-k / top-p sampling (Model.generate: decode loop)
    from zaremba_b200 import beam_step        # one on-device beam-search step (Model.beam_search: the whole search)
    from zaremba_b200 import NeuralCache      # neural-cache evaluation (Trainer.perplexity(cache=...))
    from zaremba_b200 import GradStats        # dynamic evaluation's statistics (Trainer.dynamic_perplexity)
"""
from .model import Model, Embed, LSTM, Linear  # noqa: F401
from .trainer import Trainer, minibatch  # noqa: F401
from .sampling import sample, beam_step  # noqa: F401
from .cache import NeuralCache, cache_step  # noqa: F401
from .dyneval import GradStats  # noqa: F401
from . import ensemble, parallel  # noqa: F401

__all__ = ["Model", "Embed", "LSTM", "Linear", "Trainer", "minibatch", "sample", "beam_step", "NeuralCache",
           "cache_step", "GradStats"]
