"""Crop boxes of a trained scene (DESIGN.md §3n): render, measure and extract only what lies inside a box, or everything but it.

A ``Crop`` is a box in the normalised scene frame (the frame ``Mesh`` and ``PointCloud`` are made in): the 3x4 matrix
``box_from_scene`` M maps a scene point x to the box's frame, b = M (x, 1), and the point is inside when |b_k| <= 1 for all three
k.  The kernels evaluate b_k = fma(M[k][0], x, fma(M[k][1], y, fma(M[k][2], z, M[k][3]))) in fp32 on ``box12()``, the fp32 rows
of M (csrc/crop.cuh); ``mask`` runs that predicate over points (``f2b_crop_mask``), so nothing restates it on the host.  A crop
keeps the points inside its box, or, with ``invert``, the points outside it.
"""
import numpy as np
import torch

from ._lib import call, stream

ORTHONORMAL_TOL = 1e-6


def _array(x, shape, name):
    a = np.asarray(x.detach().cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float64)
    if a.shape != shape:
        raise ValueError(f"Crop: {name} must have shape {shape}, got {a.shape}")
    if not np.isfinite(a).all():
        raise ValueError(f"Crop: {name} must be finite")
    return a


class Crop:
    """A box in the normalised scene frame and whether to keep its inside (``invert`` False) or its outside (True).
    ``box_from_scene``: [3,4] (float64 here, fp32 in the kernels) with an invertible left 3x3 block."""

    def __init__(self, box_from_scene, invert=False):
        M = _array(box_from_scene, (3, 4), "box_from_scene")
        if abs(np.linalg.det(M[:, :3])) < 1e-300:
            raise ValueError("Crop: box_from_scene must have an invertible 3x3 block")
        self.M = M
        self.invert = bool(invert)

    @classmethod
    def box(cls, bbox_min, bbox_max, invert=False, dataset=None):
        """The axis-aligned box [bbox_min, bbox_max] (scene frame, or the data's own units with ``dataset``)."""
        lo, hi = _array(bbox_min, (3,), "bbox_min"), _array(bbox_max, (3,), "bbox_max")
        return cls.oriented((lo + hi) / 2., (hi - lo) / 2., None, invert, dataset)

    @classmethod
    def oriented(cls, center, half_extents, rotation=None, invert=False, dataset=None):
        """The box center + R diag(half_extents) u, u in [-1, 1]^3: ``rotation`` R [3,3] orthonormal (its columns are the box's
        axes in the scene frame; None = identity).  With ``dataset``, the box is given in the data's own units (``in_data_frame``)."""
        c, h = _array(center, (3,), "center"), _array(half_extents, (3,), "half_extents")
        if not (h > 0).all():
            raise ValueError("Crop: every extent must be positive")
        R = np.eye(3) if rotation is None else _array(rotation, (3, 3), "rotation")
        if np.abs(R.T @ R - np.eye(3)).max() > ORTHONORMAL_TOL:
            raise ValueError(f"Crop: rotation is not orthonormal (to {ORTHONORMAL_TOL})")
        A = R.T / h[:, None]                                       # b = diag(1/h) R^T (x - c)
        crop = cls(np.concatenate([A, -(A @ c)[:, None]], 1), invert)
        return crop.in_data_frame(dataset) if dataset is not None else crop

    def in_data_frame(self, dataset):
        """This box read as one given in the data's own units -> the same box in the normalised scene frame, through
        ``load_dataset``'s normalisation x_scene = (x_data - center_) / radius_ (as ``pose.data_to_scene``)."""
        center = np.asarray(torch.as_tensor(dataset.center_).detach().cpu(), dtype=np.float64).reshape(3)
        radius = float(dataset.radius_)
        A, m = self.M[:, :3], self.M[:, 3]
        return Crop(np.concatenate([A * radius, (A @ center + m)[:, None]], 1), self.invert)

    def inverted(self):
        """The same box keeping the other side."""
        return Crop(self.M, not self.invert)

    def aabb(self):
        """(min, max) corners of the box's axis-aligned bounding box in the scene frame (of the box, whatever ``invert`` is)."""
        Ai = np.linalg.inv(self.M[:, :3])
        c = -Ai @ self.M[:, 3]
        e = np.abs(Ai).sum(1)
        return tuple(float(x) for x in c - e), tuple(float(x) for x in c + e)

    def box12(self):
        """The fp32 rows of box_from_scene the kernels take: a contiguous float32 [12] host array."""
        return np.ascontiguousarray(self.M.astype(np.float32).reshape(12))

    def mask(self, pts):
        """kept [n] bool (device) of points [n,3] (device float32, scene frame): the kernels' predicate, ``f2b_crop_mask``."""
        pts = pts.reshape(-1, 3).to(torch.float32).contiguous()
        kept = torch.empty((pts.shape[0],), dtype=torch.uint8, device=pts.device)
        box = self.box12()
        call("f2b_crop_mask", pts, int(pts.shape[0]), box.ctypes.data, int(self.invert), kept, stream())
        return kept.bool()

    def __repr__(self):
        return f"Crop(box_from_scene={self.M.tolist()}, invert={self.invert})"


def resolve_crop(crop):
    """``crop`` as the renderer takes it: None (no crop) or a ``Crop``; anything else raises ValueError."""
    if crop is not None and not isinstance(crop, Crop):
        raise ValueError(f"crop: expected None or a Crop, got {type(crop).__name__}")
    return crop
