"""H100-native hot path of neptune-ai/open-solution-mapping-challenge: ResNet-encoder U-Net forward/backward, the
weighted-CE + Dice loss and the per-pixel mask post-processing, as hand-written sm_90a CUDA behind a C ABI
(libmcb200.so, include/mcb200.h).  The Python modules mirror the reference's plugin surface:

    mcb200.unet_models.UNetResNet          <- src/unet_models.py:315-403
    mcb200.models.PyTorchUNet[Weighted]    <- src/models.py:50-209
    mcb200.postprocessing.*                <- src/postprocessing.py:48-258, src/utils.py:231-413
"""
from . import _lib  # noqa: F401  (loads libmcb200.so; raises if it is missing)

__all__ = ["_lib"]
