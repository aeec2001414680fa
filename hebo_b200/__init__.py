"""hebo_b200 -- H100-native exact-GP fit + batched MACE acquisition behind HEBO's plugin surface."""
from . import _lib  # noqa: F401
from .gp import GP, B200GP, MultiTaskModel, register  # noqa: F401
from .acq import MACE, FusedMACE, Mean, Sigma, LCB, AbsEtaDifference  # noqa: F401
from .embedding import HEBO_Embedding, MACE_Embedding  # noqa: F401
from .bo import BO, NoMR_BO, HEBO_VectorContextual  # noqa: F401
from .acq import NoisyAcq  # noqa: F401
from .noisy import NoisyOpt  # noqa: F401
from .acq import GeneralAcq, MOMeanSigmaLCB  # noqa: F401
from .general import GeneralBO  # noqa: F401

__all__ = ["GP", "B200GP", "MultiTaskModel", "MACE", "FusedMACE", "Mean", "Sigma", "LCB", "register", "HEBO_Embedding", "MACE_Embedding",
           "AbsEtaDifference", "BO", "NoMR_BO", "HEBO_VectorContextual", "NoisyOpt", "NoisyAcq",
           "GeneralAcq", "GeneralBO", "MOMeanSigmaLCB"]
