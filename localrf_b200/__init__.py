"""localrf_b200 -- H100-native (sm_90a) render path of facebookresearch/localrf.

Public surface = the reference's own module API for this path:

    from localrf_b200 import LocalTensorfs, TensorVMSplit, AlphaGridMask

backed by the C ABI in include/localrf_b200.h (localrf_b200/csrc/liblrf_b200.so).
"""
from .tensorf import AlphaGridMask, MLPRender_Fea_late_view, TensorBase, TensorVMSplit  # noqa: F401
from .local_tensorfs import LocalTensorfs, ids2pixel, ids2pixel_view  # noqa: F401
from . import data, export, losses, metrics, optim, ray_utils, utils  # noqa: F401
from .data import DeviceFrameDataset, DeviceRaySampler  # noqa: F401
from .losses import supervision_losses  # noqa: F401
from .optim import adam_step  # noqa: F401
from .pipeline import FramePipeline  # noqa: F401
from ._lib import build, lib  # noqa: F401

__version__ = "0.1.0"
