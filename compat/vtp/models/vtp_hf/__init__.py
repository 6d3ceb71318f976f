"""`vtp.models.vtp_hf` (reference: vtp/models/vtp_hf/__init__.py:18-25) served by the sm_90a implementation."""
import os
import sys

_root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))))
if _root not in sys.path:
    sys.path.insert(0, _root)

from vtp_b200.config import VTPConfig  # noqa: E402,F401
from vtp_b200.model import VTPModel, VTPPreTrainedModel  # noqa: E402,F401

__all__ = ["VTPConfig", "VTPModel", "VTPPreTrainedModel"]
