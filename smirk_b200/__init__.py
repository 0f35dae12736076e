"""smirk_b200 — H100-native implementation of SMIRK's per-frame hot path
(SmirkEncoder -> FLAME -> Renderer -> SmirkGenerator), and the trainer's VGGPerceptualLoss, MICA and ExpressionLoss,
behind the reference's class signatures.

All arithmetic runs in hand-written sm_90a CUDA (``csrc/``) behind the C ABI of
``include/smirk_b200.h``; PyTorch supplies device memory, streams and torch.distributed only.
"""
from .flame import FLAME                    # noqa: F401
from .renderer import Renderer              # noqa: F401
from .smirk_encoder import SmirkEncoder     # noqa: F401
from .smirk_generator import SmirkGenerator # noqa: F401
from .vgg_loss import VGGPerceptualLoss     # noqa: F401
from .mica import MICA                      # noqa: F401
from .expression_loss import ExpressionLoss # noqa: F401

__all__ = ["FLAME", "Renderer", "SmirkEncoder", "SmirkGenerator", "VGGPerceptualLoss", "MICA", "ExpressionLoss"]
__version__ = "0.1.0"
