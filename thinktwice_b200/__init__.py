"""thinktwice_b200 — H100-native implementation of the ThinkTwice per-frame forward path.

Importing the package registers the boundary classes (EncoderDecoder, LSS, LidarNet, SparseEncoder_fp32,
ThinkTwiceDecoder) exactly like the reference's plugin import does (open_loop_training/code/__init__.py).
"""
__version__ = '0.1.0'

from .registry import (BACKBONES, DETECTORS, HEADS, MIDDLE_ENCODERS, NECKS, build_backbone, build_head,  # noqa: F401
                       build_model, register_into_mmdet)
from .encoder_decoder_framework import EncoderDecoder  # noqa: F401,E402
from .lss import LSS  # noqa: F401,E402
from .lidarnet import LidarNet, SparseEncoder_fp32  # noqa: F401,E402
from .thinktwice_decoder import ThinkTwiceDecoder  # noqa: F401,E402

register_into_mmdet()
