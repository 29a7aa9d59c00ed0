"""Lenses for views of a trained scene (DESIGN.md §3o): equirectangular panoramas, omnidirectional-stereo (ODS) pairs, equidistant
fisheye views and pinhole views of any size and field of view.

A ``Lens`` makes the rays of one image through a camera pose: ``f2b_lens_rays`` (csrc/rays.cu) for the panoramic and fisheye
models, ``f2b_camera_rays`` with undistorted intrinsics for the pinhole.  ``eval.RenderLens`` renders them; ``level_pose`` gives
a pose whose "up" is the training cameras' mean up, which panoramas of scenes reconstructed in an arbitrary frame need.
"""
import math

import numpy as np
import torch

from ._lib import call, stream

PINHOLE, EQUIRECT, FISHEYE, ODS = "pinhole", "equirect", "fisheye", "ods"
_MODEL = {EQUIRECT: 0, FISHEYE: 1, ODS: 2}            # F2B_LENS_* (include/f2nerf_b200.h)
_MAX_RAYS = 1 << 31


def _size(v, name):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or int(v) < 1:
        raise ValueError(f"Lens: {name} must be an integer >= 1, got {v!r}")
    return int(v)


def _angle(v, name, hi, hi_open=False):
    v = float(v)
    if not math.isfinite(v) or v <= 0. or v > hi or (hi_open and v == hi):
        raise ValueError(f"Lens: {name} must be in (0, {hi}{')' if hi_open else ']'} degrees, got {v}")
    return v


def _pose64(pose):
    p = torch.as_tensor(np.asarray(pose.detach().cpu() if isinstance(pose, torch.Tensor) else pose, dtype=np.float64))
    if p.shape != (3, 4):
        raise ValueError(f"Lens: a pose is [3,4] (camera to world), got shape {tuple(p.shape)}")
    if not bool(torch.isfinite(p).all()):
        raise ValueError("Lens: the pose must be finite")
    return p


class Lens:
    """One image's camera model and size.  Build it with ``pinhole``, ``equirect``, ``fisheye`` or ``ods``; ``shape`` is the
    image's (height, width), 2H x W for an ODS pair (left eye on top)."""

    def __init__(self, model, height, width, p0, p1=0., p2=0.):
        self.model, self.height, self.width = model, height, width
        self.p0, self.p1, self.p2 = float(p0), float(p1), float(p2)
        if self.n_rays >= _MAX_RAYS:
            raise ValueError(f"Lens: {self.shape[0]} x {self.shape[1]} rays overflow int32")

    @classmethod
    def pinhole(cls, height, width, vfov):
        """A distortion-free pinhole with square pixels: fx = fy = (H / 2) / tan(vfov / 2), principal point (W / 2, H / 2)."""
        return cls(PINHOLE, _size(height, "height"), _size(width, "width"), _angle(vfov, "vfov", 180., hi_open=True))

    @classmethod
    def equirect(cls, height, width=None, hfov=360., vfov=180.):
        """An equirectangular image: longitude linear in the column over hfov, latitude linear in the row over vfov (a VR180
        image is hfov = vfov = 180).  ``width`` defaults to 2 * height."""
        h = _size(height, "height")
        return cls(EQUIRECT, h, _size(2 * h if width is None else width, "width"), _angle(hfov, "hfov", 360.),
                   _angle(vfov, "vfov", 180.))

    @classmethod
    def fisheye(cls, height, width=None, fov=180.):
        """An equidistant fisheye (angle to the axis proportional to the distance from the centre) whose circle of ``fov`` degrees
        (up to 360) fills min(height, width); pixels outside it are not valid.  ``width`` defaults to ``height``."""
        h = _size(height, "height")
        return cls(FISHEYE, h, _size(h if width is None else width, "width"), _angle(fov, "fov", 360.))

    @classmethod
    def ods(cls, height, width=None, hfov=360., vfov=180., ipd=0.064):
        """An omnidirectional-stereo pair: two equirectangular images (left eye on top), each eye on a circle of diameter ``ipd``
        around the pose's position, offset at right angles to each column's viewing direction.  ``ipd`` is in scene units, or in
        the data's own units when the rays are made with a dataset."""
        h = _size(height, "height")
        ipd = float(ipd)
        if not math.isfinite(ipd) or ipd < 0.:
            raise ValueError(f"Lens: ipd must be finite and >= 0, got {ipd}")
        return cls(ODS, h, _size(2 * h if width is None else width, "width"), _angle(hfov, "hfov", 360.), _angle(vfov, "vfov", 180.),
                   ipd)

    @property
    def shape(self):
        return (2 * self.height if self.model == ODS else self.height, self.width)

    @property
    def n_rays(self):
        return self.shape[0] * self.shape[1]

    @property
    def may_be_invalid(self):
        """Whether some pixels have no ray (outside a fisheye's circle)."""
        return self.model == FISHEYE

    def intrinsics(self):
        """The pinhole's K [3,3] float64 (numpy)."""
        if self.model != PINHOLE:
            raise ValueError(f"Lens: a {self.model} lens has no pinhole intrinsics")
        f = (self.height / 2.) / math.tan(math.radians(self.p0) / 2.)
        return np.array([[f, 0., self.width / 2.], [0., f, self.height / 2.], [0., 0., 1.]])

    def rays(self, pose, dataset=None, device=None):
        """-> device (rays_o [N,3], rays_d [N,3], valid [N] bool), ray a * W + b through the centre of pixel (a, b) of ``shape``.
        ``pose``: [3,4] camera to world in the normalised scene frame, or with ``dataset`` in the data's own frame (then the ipd too
        is in data units).  Directions are not normalised (the renderer normalises them); rays_d = 0 where not valid."""
        p = _pose64(pose)
        p2 = self.p2
        if dataset is not None:
            from .pose import data_to_scene
            p = data_to_scene(p, dataset)
            p2 = p2 / float(dataset.radius_)
            dev = dataset.poses_.device if device is None else torch.device(device)
        else:
            dev = torch.device("cuda" if device is None else device)
        p32 = p.to(torch.float32).to(dev).contiguous()
        n = self.n_rays
        rays_o = torch.empty((n, 3), dtype=torch.float32, device=dev)
        rays_d = torch.empty((n, 3), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if self.model == PINHOLE:
                K = torch.from_numpy(self.intrinsics()).to(torch.float32).to(dev).contiguous()
                dist = torch.zeros((4,), dtype=torch.float32, device=dev)
                call("f2b_camera_rays", p32, K, dist, self.height, self.width, self.height, self.width, rays_o, rays_d, stream())
                return rays_o, rays_d, torch.ones((n,), dtype=torch.bool, device=dev)
            valid = torch.empty((n,), dtype=torch.uint8, device=dev)
            call("f2b_lens_rays", _MODEL[self.model], p32, self.height, self.width, self.p0, self.p1, p2, rays_o, rays_d, valid,
                 stream())
        return rays_o, rays_d, valid.view(torch.bool)

    def __repr__(self):
        args = {PINHOLE: f"vfov={self.p0}", EQUIRECT: f"hfov={self.p0}, vfov={self.p1}", FISHEYE: f"fov={self.p0}",
                ODS: f"hfov={self.p0}, vfov={self.p1}, ipd={self.p2}"}[self.model]
        return f"Lens.{self.model}({self.height}, {self.width}, {args})"


def _unit(v, what):
    n = float(torch.linalg.norm(v))
    if not n > 1e-12:
        raise ValueError(f"level_pose: the training cameras' mean {what} is zero")
    return v / n


def _rot(axis, deg):
    """Rodrigues: the rotation by ``deg`` degrees about the unit ``axis`` (float64)."""
    x, y, z = (float(c) for c in axis)
    K = torch.tensor([[0., -z, y], [z, 0., -x], [-y, x, 0.]], dtype=torch.float64)
    a = math.radians(deg)
    return torch.eye(3, dtype=torch.float64) + math.sin(a) * K + (1. - math.cos(a)) * (K @ K)


def level_pose(dataset, position, yaw_deg=0., pitch_deg=0.):
    """A level camera pose [3,4] (float64, CPU, camera to world in the normalised scene frame).  Its +y is the normalised mean
    of the training cameras' up columns; its -z the training cameras' mean forward (-z column) with the up component removed,
    turned by ``yaw_deg`` about up (positive towards the camera's right) and then by ``pitch_deg`` about its x axis (positive
    looks up; the camera's y tilts with it).  ``position``: a scene-frame point [3], or an int, the index of a camera whose
    position is taken."""
    yaw, pitch = float(yaw_deg), float(pitch_deg)
    if not (math.isfinite(yaw) and math.isfinite(pitch)):
        raise ValueError("level_pose: yaw and pitch must be finite")
    poses = dataset.poses_.detach().to("cpu", torch.float64)
    train = list(dataset.train_set_) or list(range(poses.shape[0]))
    rot = poses[train, :, :3]
    up = _unit(rot[:, :, 1].mean(0), "up")
    fwd = -rot[:, :, 2].mean(0)
    fwd = _unit(fwd - (fwd @ up) * up, "forward (off up)")
    if isinstance(position, (int, np.integer)) and not isinstance(position, bool):
        if not 0 <= int(position) < poses.shape[0]:
            raise ValueError(f"level_pose: camera {position} outside [0, {poses.shape[0]})")
        t = poses[int(position), :, 3]
    else:
        t = torch.as_tensor(np.asarray(position.detach().cpu() if isinstance(position, torch.Tensor) else position, dtype=np.float64))
        if t.shape != (3,) or not bool(torch.isfinite(t).all()):
            raise ValueError(f"level_pose: position must be a finite point [3] or a camera index, got {position!r}")
    fwd = _rot(up, -yaw) @ fwd                                    # about +y, a positive angle turns -z towards -x: negate
    z = -fwd
    x = torch.linalg.cross(up, z)
    R = torch.stack([x, up, z], 1)
    R = R @ _rot(torch.tensor([1., 0., 0.]), pitch)                # about the camera's x: positive turns -z towards +y
    return torch.cat([R, t[:, None]], 1)
