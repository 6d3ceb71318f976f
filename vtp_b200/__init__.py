"""vtp_b200 — H100-native (sm_90a) implementation of the MiniMax-AI/VTP hot path behind the reference's own API."""
from .config import VTPConfig, preset  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not require torch.cuda
    if name in ("VTPModel", "VTPPreTrainedModel"):
        from . import model
        return getattr(model, name)
    if name in ("VTPTrainer", "TrainConfig"):
        from . import train
        return getattr(train, name)
    raise AttributeError(name)
