"""f2nerf_b200 — H100-native (sm_90a) implementation of F2-NeRF's per-ray rendering hot path.

The product is ``libf2nerf_b200.so`` (hand-written CUDA behind the C ABI in ``include/f2nerf_b200.h``);
this package is the thin host-side mirror of the reference's operator surface
(``PersSampler`` / ``Hash3DAnchored`` / ``TCNNWP`` / ``SHShader`` / ``Renderer`` / ``FlexOps`` /
``CustomOps``) that feeds it device pointers.  Importing it without the built library raises.
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA extension is missing)
from .appearance import FitAppearance, TestAppearance
from .crop import Crop
from .checkpoint import Scene, gradient_scaling_progress, load_scene, load_states
from .dataset import RayGenerator, load_dataset
from .octree_build import build_edge_pool, build_tree_nodes, initial_octree
from .eval import ImageMetrics, RenderAllImages, RenderDepth, RenderLens, RenderNormals, RenderPath, RenderWholeImage, TestImages
from .field import Hash3DAnchored, TCNNWP
from .geometry import ExtractTSDFMesh, FuseTSDF, TSDFGrid, TSDFSurface
from .lens import Lens, level_pose
from .ops import CustomOps, FlexOps
from .optim import FusedAdam
from .pose import RayGradient, RefinePose
from .renderer import Renderer, RenderResult, check_backward_nan
from .sampler import TRAIN, VALIDATE, GlobalDataPool, PersSampler, SampleResultFlex
from .shader import SHShader

__all__ = ["ExtractTSDFMesh", "FuseTSDF", "TSDFGrid", "TSDFSurface", "Crop", "Lens", "level_pose", "RenderLens", "FitAppearance", "TestAppearance", "FusedAdam", "RayGradient", "RefinePose", "RayGenerator", "load_dataset", "load_scene", "load_states", "Scene", "gradient_scaling_progress",
           "build_tree_nodes", "build_edge_pool", "initial_octree", "RenderWholeImage", "RenderDepth", "RenderNormals", "TestImages", "ImageMetrics", "RenderPath", "RenderAllImages", "Hash3DAnchored", "TCNNWP", "CustomOps", "FlexOps", "Renderer", "RenderResult", "check_backward_nan",
           "TRAIN", "VALIDATE", "GlobalDataPool", "PersSampler", "SampleResultFlex", "SHShader"]
