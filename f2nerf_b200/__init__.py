"""f2nerf_b200 — H100-native (sm_90a) implementation of F2-NeRF's per-ray rendering hot path.

The product is ``libf2nerf_b200.so`` (hand-written CUDA behind the C ABI in ``include/f2nerf_b200.h``);
this package is the thin host-side mirror of the reference's operator surface
(``PersSampler`` / ``Hash3DAnchored`` / ``TCNNWP`` / ``SHShader`` / ``Renderer`` / ``FlexOps`` /
``CustomOps``) that feeds it device pointers.  Importing it without the built library raises.
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA extension is missing)
from .dataset import RayGenerator
from .eval import ImageMetrics, RenderAllImages, RenderPath, RenderWholeImage, TestImages
from .field import Hash3DAnchored, TCNNWP
from .ops import CustomOps, FlexOps
from .optim import FusedAdam
from .renderer import Renderer, RenderResult, check_backward_nan
from .sampler import TRAIN, VALIDATE, GlobalDataPool, PersSampler, SampleResultFlex
from .shader import SHShader

__all__ = ["FusedAdam", "RayGenerator", "RenderWholeImage", "TestImages", "ImageMetrics", "RenderPath", "RenderAllImages", "Hash3DAnchored", "TCNNWP", "CustomOps", "FlexOps", "Renderer", "RenderResult", "check_backward_nan",
           "TRAIN", "VALIDATE", "GlobalDataPool", "PersSampler", "SampleResultFlex", "SHShader"]
