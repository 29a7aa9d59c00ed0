"""Camera poses against a trained scene (DESIGN.md §3k): the gradient of the rendered colour with respect to its rays, and the
refinement of a camera pose from a photo of the scene.

``RayGradient`` renders a batch as the VALIDATE ``Render`` does (``f2b_render_phase1`` + ``f2b_render_phase2_fwd``, no edge points,
colours bit-identical to ``Renderer.render_forward``) and pulls a dL/dcolors back to the ray origins and directions through the
composite, shader-MLP and shading-input backward and ``f2b_ray_grad``.  The sample distances t, dt, the kept samples and their
leaves are held fixed, as NeRF pose-refinement methods hold them.  Nothing of the scene is written: no octree votes, no statistics,
no draw from the default CUDA generator, and ``Renderer.sample_result_`` is left alone (the march runs in buffers of its own).

``RefinePose`` fits the 6-vector xi of ``pose = exp(xi) o pose0`` (Rodrigues rotation, then translation; float64 on the host) to a
photo with Adam on the mean squared colour error of ``n_rays`` pixels drawn per iteration from a seeded host generator.
"""
import math

import numpy as np
import torch

from . import _lib, ops
from ._lib import call, stream
from .eval import _Validate
from .sampler import MAX_SAMPLE_PER_RAY

F64 = torch.float64
# Loss scales of the backward chain (powers of two, so un-scaling is exact).  A photometric loss over a few thousand rays gives
# dL/dcolors of ~1e-4; the trainer's 128 leaves most fp16 rows subnormal there (DESIGN.md §3k has the measured fractions).
SHADER_LOSS_SCALE = 2. ** 20
FIELD_LOSS_SCALE = 2. ** 20
_MAX_BACKOFF = 12


# ------------------------------------------------------------------------------------------------------------------- the ray VJP
class _Batch:
    """The forward of one ray batch and every buffer the backward reads."""


def _render(renderer, rays_o, rays_d_unit, app=None):
    """VALIDATE render of unit-direction rays through the launch sequences: march into own scratch, early stop, compaction, field,
    shader, composite.  One host sync (the survivor count).  ``app``: an appearance row [16] for every ray, through phase 2's
    embedding path (a [1,16] table, every ray on row 0)."""
    field, shader, sampler = renderer.scene_field_, renderer.shader_, renderer.pts_sampler_
    R, dev = rays_o.shape[0], rays_o.device
    S = MAX_SAMPLE_PER_RAY
    i32 = lambda *sh: torch.empty(sh, dtype=torch.int32, device=dev)
    f16 = lambda *sh: torch.empty(sh, dtype=torch.float16, device=dev)
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
    b = _Batch()
    b.renderer, b.n_rays, b.rays_o = renderer, R, rays_o
    with _Validate(renderer):
        b.noise = sampler.make_noise(R, dev)                     # VALIDATE: ones * fineness, no draw
        b.bg = renderer._bg(R, dev)                              # VALIDATE: no draw
    b.table16 = field.table_f16()
    b.fparams16, b.sparams16 = f16(field.mlp_.params_.numel()), f16(shader.mlp_.params_.numel())
    b.new_bounds, heads = i32(R, 2), i32(3)
    b.march_counts, b.kept_counts = i32(R), i32(R)
    ra = _lib.RenderArgs()
    ra.set(tree_nodes=sampler.tree_nodes_gpu_, n_nodes=sampler.n_nodes, trans=sampler.pers_trans_gpu_,
           n_trans=sampler.pers_trans_gpu_.numel() // 544, edge_pool=None, near_t=float(sampler.global_near_), far_t=1e8,
           sample_l=float(sampler.sample_l_), scale_by_dis=int(sampler.scale_by_dis_), max_hits=int(sampler.max_oct_intersect_per_ray_),
           count_all_hits=0, table16=b.table16, prim=field.prim_pool_, bias=field.bias_pool_, n_volumes=int(field.n_volumes_),
           local_size=int(field.local_size_), field_params=field.mlp_.params_.detach(), n_field_params=b.fparams16.numel(),
           shader_params=shader.mlp_.params_.detach(), n_shader_params=b.sparams16.numel(), fparams16=b.fparams16,
           sparams16=b.sparams16, n_rays=R, rays_o=rays_o, rays_d=rays_d_unit, noise=b.noise, bg=b.bg, skip_march=0,
           counts=b.march_counts, totals=heads[1:], kept_counts=b.kept_counts, new_bounds=b.new_bounds, total_kept=heads, stream=stream())
    # the argument block holds raw pointers: every buffer it points to stays referenced from the batch
    b.scratch = dict(s_pts=f32(R * S, 3), s_dt=f32(R * S), s_t=f32(R * S), s_anchors=i32(R * S, 2), chunk_bounds=i32(R, 2),
                     slot_bounds=i32(R, 2), first_oct_dis=f32(R, 1), logit_s=f32(R * S), feat_s=f16(R * S, 32), w0=f32(R * S),
                     a0=f32(R * S), keep=torch.empty((R * S,), dtype=torch.uint8, device=dev))
    ra.set(**b.scratch)
    b.keep_alive = [rays_o, rays_d_unit, heads, ra]
    if app is not None:
        b.app_table, b.ray_emb_idx = app.reshape(1, 16).contiguous(), torch.zeros((R,), dtype=torch.int32, device=dev)
        ra.set(app_emb=b.app_table, n_emb=1, ray_emb_idx=b.ray_emb_idx)
    call("f2b_render_phase1", ra)
    n_kept, n_all, _ = heads.tolist()
    b.n_kept, b.n_all = n_kept, n_all
    if n_all <= 0:                                               # the reference's empty-batch result (Renderer.cpp:83-97)
        b.colors = b.bg.clone()
        return b
    T = dict(pts=f32(n_kept, 3), dirs=f32(n_kept, 3), dt=f32(n_kept), t=f32(n_kept), anchors=i32(n_kept, 3), feat_q=f16(n_kept, 32),
             logit=f32(n_kept), mlp_in=f16(n_kept, 32), raw=f16(n_kept, 16), rgb=f32(n_kept, 3), colors=f32(R, 3),
             disparity=f32(R), depth=f32(R), weights=f32(n_kept))
    if app is not None:
        T["pt_emb_idx"] = i32(n_kept)
    ra.set(n_kept=n_kept, n_edge_pairs=0, **T)
    call("f2b_render_phase2_fwd", ra)
    b.T, b.ra = T, ra
    b.colors = T["colors"]
    return b


def _shader_input_bwd(b, d_colors, shader_scale):
    """dL/dcolors -> (d_logit [P'], d_raw [P',16], d_in16 [P',32]) of the kept samples: the composite and colour-activation backward
    and the shader MLP's backward to its input rows.  d_raw and d_in16 are fp16 and scaled by ``shader_scale``."""
    nk, T, dev = b.n_kept, b.T, b.rays_o.device
    d_colors = d_colors.to(device=dev, dtype=torch.float32).contiguous()
    d_logit = torch.empty((nk,), dtype=torch.float32, device=dev)
    d_raw, d_in16 = (torch.empty((nk, c), dtype=torch.float16, device=dev) for c in (16, 32))
    d_sparams = torch.zeros((b.sparams16.numel(),), dtype=torch.float32, device=dev)       # scratch: the scene is not trained
    if nk > 0:
        call("f2b_composite_act_bwd", T["logit"], 1, T["rgb"], T["dt"], T["t"], b.new_bounds, b.bg, b.n_rays, d_colors, None, None, None,
             1.0, T["raw"], float(shader_scale), d_logit, 1, d_raw, stream())
        call("f2b_mlp_bwd2", d_raw, T["mlp_in"], None, None, b.sparams16, 1, nk, d_in16, d_sparams, stream())
    return d_logit, d_raw, d_in16


def _backprop(b, d_colors, shader_scale, field_scale, rows=False):
    """dL/dcolors -> (d_o [R,3], d_dhat [R,3]) with respect to the origins and the unit directions; ``rows``: also the per-row
    tensors of the chain (tests, probe)."""
    R, dev = b.n_rays, b.rays_o.device
    d_o = torch.zeros((R, 3), dtype=torch.float32, device=dev)
    d_d = torch.zeros((R, 3), dtype=torch.float32, device=dev)
    out = dict(d_o=d_o, d_d=d_d)
    if b.n_all <= 0:
        return out
    nk, T, f = b.n_kept, b.T, b.renderer.scene_field_
    f16 = lambda *sh: torch.empty(sh, dtype=torch.float16, device=dev)
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
    d_logit, d_raw, d_in16 = _shader_input_bwd(b, d_colors, shader_scale)
    d_out16 = f16(nk, 16)
    work = f32(max(nk, 1), 6)
    d_pts = f32(nk, 3) if rows else None
    d_dirs = f32(nk, 3) if rows else None
    dfeat16 = f16(nk, 32) if rows else None
    if nk > 0:
        ops.shader_prep_bwd_f16(d_in16, d_logit, b.new_bounds, None, 1.0 / shader_scale, float(field_scale), d_out16, None)
    ops.ray_grad(b.renderer.pts_sampler_.pers_trans_gpu_, b.table16, f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_,
                 b.fparams16, T["feat_q"], d_out16, d_in16, T["pts"], T["t"], T["dirs"], T["anchors"], b.rays_o, b.new_bounds,
                 1.0 / field_scale, 1.0 / shader_scale, work, d_o, d_d, d_pts, d_dirs, dfeat16)
    if rows:
        out.update(d_logit=d_logit, d_raw=d_raw, d_in16=d_in16, d_field_out=d_out16, d_pts=d_pts, d_dirs=d_dirs, dfeat16=dfeat16,
                   **{k: T[k] for k in ("pts", "dirs", "dt", "t", "anchors", "feat_q", "logit", "mlp_in", "raw", "rgb", "weights")},
                   new_bounds=b.new_bounds, bg=b.bg, n_kept=nk, march_counts=b.march_counts, kept_counts=b.kept_counts)
    return out


def _chain_normalise(rays_d, d_dhat):
    """dL/dd from dL/dd^ for d^ = d / |d| (PersSampler.cu:319): (dL/dd^ - d^ (d^ . dL/dd^)) / |d|."""
    n = torch.linalg.norm(rays_d, 2, -1, True)
    dh = rays_d / n
    return (d_dhat - dh * (dh * d_dhat).sum(-1, keepdim=True)) / n


def _unit(rays_d):
    return (rays_d / torch.linalg.norm(rays_d, 2, -1, True)).contiguous()


def backed_off(backward, finite, what):
    """``backward(shader_scale, field_scale)`` at the fixed loss scales, backed off (both halved, as the trainer halves its scale)
    only while ``finite(out)`` is False -> (out, shader_scale, field_scale)."""
    sh, fs = SHADER_LOSS_SCALE, FIELD_LOSS_SCALE
    for _ in range(_MAX_BACKOFF):
        out = backward(sh, fs)
        if finite(out):
            return out, sh, fs
        sh, fs = max(sh / 2., 1.), max(fs / 2., 1.)
    raise FloatingPointError(f"{what} at every loss scale")


def _vjp(b, d_colors, rays_d, rows=False):
    """Backward at the fixed loss scales, backed off (both halved, as the trainer halves its scale) only while the gradients are
    not finite."""
    out, sh, fs = backed_off(lambda sh, fs: _backprop(b, d_colors, sh, fs, rows),
                             lambda out: bool(torch.isfinite(out["d_o"]).all() & torch.isfinite(out["d_d"]).all()),
                             "RayGradient: non-finite ray gradients")
    d_dhat = out["d_d"]
    out.update(d_dhat=d_dhat, d_d=_chain_normalise(rays_d, d_dhat), shader_loss_scale=sh, field_loss_scale=fs)
    return out


def _check_rays(rays_o, rays_d, dev):
    if rays_o.ndim != 2 or rays_o.shape[1] != 3 or rays_d.shape != rays_o.shape:
        raise ValueError(f"RayGradient: rays_o and rays_d must both be [R,3], got {tuple(rays_o.shape)} and {tuple(rays_d.shape)}")
    return (rays_o.to(device=dev, dtype=torch.float32).contiguous(), rays_d.to(device=dev, dtype=torch.float32).contiguous())


def RayGradient(renderer, rays_o, rays_d, d_colors, rows=False):
    """-> (colors [R,3], dL/drays_o [R,3], dL/drays_d [R,3]) for the raw directions ``rays_d`` (the sampler's normalisation is
    part of the VJP).  ``colors`` are bit-identical to the VALIDATE ``Render``'s; the gradients have the same bits on every run
    and for any split of the batch.  ``rows=True`` returns a dict with the per-sample tensors of the chain instead."""
    dev = renderer.app_emb_.device
    rays_o, rays_d = _check_rays(rays_o, rays_d, dev)
    if d_colors.shape != rays_o.shape:
        raise ValueError(f"RayGradient: d_colors must be [R,3] like the rays, got {tuple(d_colors.shape)}")
    with torch.no_grad():
        b = _render(renderer, rays_o, _unit(rays_d))
        out = _vjp(b, d_colors.to(device=dev, dtype=torch.float32), rays_d, rows)
    if rows:
        out["colors"] = b.colors
        return out
    return b.colors, out["d_o"], out["d_d"]


class RayColors(torch.autograd.Function):
    """colors = render(rays_o, rays_d) with ``RayGradient``'s VJP as its backward (the scene's parameters take no gradient)."""

    @staticmethod
    def forward(ctx, rays_o, rays_d, renderer):
        dev = renderer.app_emb_.device
        o, d = _check_rays(rays_o.detach(), rays_d.detach(), dev)
        b = _render(renderer, o, _unit(d))
        ctx.batch, ctx.rays_d = b, d
        return b.colors.clone()

    @staticmethod
    def backward(ctx, d_colors):
        out = _vjp(ctx.batch, d_colors.contiguous(), ctx.rays_d)
        ctx.batch = None
        return out["d_o"], out["d_d"], None


# ----------------------------------------------------------------------------------------------------------- pose parameterisation
def _as64(x):
    return x if isinstance(x, torch.Tensor) and x.dtype == F64 and x.device.type == "cpu" else torch.as_tensor(np.asarray(
        x.detach().cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float64))


def so3_exp(w):
    """Rodrigues: the rotation [3,3] of the axis-angle 3-vector ``w`` (float64, differentiable; the second-order series near 0)."""
    th2 = (w * w).sum()
    K = torch.zeros((3, 3), dtype=w.dtype, device=w.device)
    K = K.index_put((torch.tensor([0, 0, 1, 1, 2, 2]), torch.tensor([1, 2, 0, 2, 0, 1])),
                    torch.stack([-w[2], w[1], w[2], -w[0], -w[1], w[0]]))
    if float(th2.detach()) < 1e-12:
        a, c = 1. - th2 / 6., .5 - th2 / 24.
    else:
        th = torch.sqrt(th2)
        a, c = torch.sin(th) / th, (1. - torch.cos(th)) / th2
    return torch.eye(3, dtype=w.dtype, device=w.device) + a * K + c * (K @ K)


def se3_exp(xi):
    """The rigid transform [3,4] of the 6-vector xi = (axis-angle w, translation v): [so3_exp(w) | v]."""
    xi = xi if isinstance(xi, torch.Tensor) else torch.as_tensor(xi, dtype=F64)
    if xi.shape != (6,):
        raise ValueError(f"se3_exp: xi must have 6 entries, got shape {tuple(xi.shape)}")
    return torch.cat([so3_exp(xi[:3]), xi[3:, None]], 1)


def compose(a, b):
    """a o b of two [3,4] camera-to-world transforms: x -> a(b(x))."""
    return torch.cat([a[:, :3] @ b[:, :3], (a[:, :3] @ b[:, 3:] + a[:, 3:])], 1)


def _check_pose(pose, what):
    p = _as64(pose)
    if p.shape != (3, 4):
        raise ValueError(f"{what}: a pose is [3,4] (camera to world), got shape {tuple(p.shape)}")
    return p


def data_to_scene(pose, dataset):
    """A camera-to-world pose [3,4] in the data's own frame -> the normalised scene frame: translation (t - center_) / radius_
    (load_dataset's NormalizeScene; the rotation is unchanged).  float64."""
    p = _check_pose(pose, "data_to_scene").clone()
    c = torch.as_tensor(np.asarray(torch.as_tensor(dataset.center_).cpu(), dtype=np.float64))
    p[:, 3] = (p[:, 3] - c) / float(dataset.radius_)
    return p


def scene_to_data(pose, dataset):
    """The inverse of ``data_to_scene``: translation t * radius_ + center_ (as ``Mesh.to_data_frame`` moves points).  float64."""
    p = _check_pose(pose, "scene_to_data").clone()
    c = torch.as_tensor(np.asarray(torch.as_tensor(dataset.center_).cpu(), dtype=np.float64))
    p[:, 3] = p[:, 3] * float(dataset.radius_) + c
    return p


def rotation_error_deg(a, b):
    """Angle in degrees of the relative rotation between two poses [3,4]."""
    r = _as64(a)[:, :3].T @ _as64(b)[:, :3]
    return math.degrees(math.acos(max(-1., min(1., (float(torch.trace(r)) - 1.) / 2.))))


def translation_error(a, b):
    return float(torch.linalg.norm(_as64(a)[:, 3] - _as64(b)[:, 3]))


def perturb(pose, angle_deg, distance, seed):
    """pose rotated by ``angle_deg`` about a seeded random axis through the camera and moved by ``distance`` in a seeded random
    direction (camera-to-world; both in the pose's frame).  float64."""
    g = np.random.default_rng(seed)
    axis, step = g.normal(size=3), g.normal(size=3)
    axis, step = axis / np.linalg.norm(axis), step / np.linalg.norm(step)
    p = _check_pose(pose, "perturb")
    R = so3_exp(torch.as_tensor(axis * math.radians(angle_deg)))
    return torch.cat([R @ p[:, :3], p[:, 3:] + torch.as_tensor(step * distance)[:, None]], 1)


# --------------------------------------------------------------------------------------------------------------- rays of a camera
def camera_directions(intri, dist_params, height, width, device="cuda"):
    """Camera-frame directions [H*W,3] of every pixel, f2b_camera_rays at the identity pose (ray a*W + b through pixel (a, b),
    undistorted with ``dist_params``).  They depend on the pixel only, so a pose moves them by one rotation."""
    dev = torch.device(device)
    f = lambda t, n: torch.as_tensor(np.asarray(t.detach().cpu() if isinstance(t, torch.Tensor) else t, dtype=np.float32)).reshape(n).to(dev).contiguous()
    K, D = f(intri, (3, 3)), f(dist_params, (4,))
    eye = torch.eye(3, 4, dtype=torch.float32, device=dev).contiguous()
    n = int(height) * int(width)
    o = torch.empty((n, 3), dtype=torch.float32, device=dev)
    d = torch.empty((n, 3), dtype=torch.float32, device=dev)
    call("f2b_camera_rays", eye, K, D, int(height), int(width), int(height), int(width), o, d, stream())
    return d


def rays_from_pose(pose, dirs_cam):
    """Rays of the camera-frame directions ``dirs_cam`` [n,3] (device) under the pose [3,4] (camera to world, scene frame):
    d = R . d_cam, o = t, differentiable with respect to the pose.  They equal RaysFromPose's rays up to fp32 rounding, not bit for
    bit (the reference forms R . d_cam in its own order)."""
    p = pose.to(device=dirs_cam.device, dtype=torch.float32)
    d = dirs_cam @ p[:, :3].T
    o = p[:, 3][None, :].expand(d.shape[0], 3)
    return o, d


def _camera(camera, dataset, height, width, what="RefinePose"):
    if isinstance(camera, (int, np.integer)):
        if dataset is None:
            raise ValueError(f"{what}: a camera given by index needs the dataset")
        i = int(camera)
        if not 0 <= i < dataset.n_images_:
            raise ValueError(f"{what}: camera index {i} outside [0, {dataset.n_images_})")
        if (dataset.height_, dataset.width_) != (height, width):
            raise ValueError(f"{what}: the image is {height}x{width}, the dataset's cameras {dataset.height_}x{dataset.width_}")
        return dataset.intri_[i], dataset.dist_params_[i]
    if not isinstance(camera, (tuple, list)) or len(camera) != 2:
        raise ValueError(f"{what}: camera is (intrinsics [3,3], distortion [4]) or a dataset index")
    return camera


def RefinePose(renderer, image, camera, pose0, iters=300, n_rays=4096, lr=2e-3, seed=0, dataset=None):
    """Refine the camera-to-world pose ``pose0`` [3,4] (normalised scene frame) of the photo ``image`` [H,W,3] (values in [0,1]).
    ``camera``: (intrinsics [3,3], distortion [4]) of the photo, or the index of a dataset camera whose intrinsics to use.
    Per iteration ``n_rays`` pixels are drawn from a ``torch.Generator`` seeded with ``seed``, the VALIDATE render of their rays is
    compared with the photo (mean squared error) and Adam (``lr``) steps xi of ``pose = exp(xi) o pose0``.  The scene's parameters and
    state are never written.  -> (pose [3,4] float64, per-iteration losses list)."""
    if iters < 0 or n_rays <= 0:
        raise ValueError(f"RefinePose: iters >= 0 and n_rays > 0 required, got {iters}, {n_rays}")
    img = torch.as_tensor(image)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"RefinePose: image must be [H,W,3], got {tuple(img.shape)}")
    H, W = int(img.shape[0]), int(img.shape[1])
    p0 = _check_pose(pose0, "RefinePose")
    intri, dist = _camera(camera, dataset, H, W)
    dev = renderer.app_emb_.device
    gt = img.to(device=dev, dtype=torch.float32).reshape(-1, 3)
    dirs = camera_directions(intri, dist, H, W, dev)
    gen = torch.Generator(device="cpu").manual_seed(int(seed))
    xi = torch.zeros(6, dtype=F64, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=lr)
    losses = []
    for _ in range(int(iters)):
        pix = torch.randint(H * W, (int(n_rays),), generator=gen).to(dev)
        pose = compose(se3_exp(xi), p0)
        o, d = rays_from_pose(pose, dirs[pix])
        colors = RayColors.apply(o.contiguous(), d.contiguous(), renderer)
        loss = ((colors - gt[pix]) ** 2).mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        pose = compose(se3_exp(xi.detach()), p0)
    return pose, losses
