"""Whole-image evaluation — SURVEY §8(f) N4: ``ExpRunner::RenderWholeImage`` (src/ExpRunner.cpp:257-293) and the three
evaluation modes built on it, ``TestImages`` (:343-391), ``RenderPath`` (:322-341) and ``RenderAllImages`` /
``VisualizeImage`` (:295-320).

The reference renders an image in fixed chunks of 8192 rays: every chunk is copied host->device, rendered
(``Renderer::Render`` in VALIDATE mode under a NoGradGuard), and three results are copied device->host and written
into CPU tensors with ``index_put_`` — 3 blocking H2D + 3 blocking D2H copies and several ``.item()``-style syncs per
chunk.  Same chunking and the same returned tensors here (CPU ``pred_colors [N,3]``, ``first_oct_disp [N,1]``,
``pred_disp [N,1]`` with the reference's normalisations), but the rays are uploaded once (pinned, asynchronous), the
per-chunk results are written straight into device-resident images, and there is ONE device->host copy at the end.
Each chunk is the march + ONE fused kernel (``Renderer.render_forward`` -> ``f2b_render_fwd_fused``, csrc/fused_fwd.cu) writing its
rows of the image; chunks alternate between two streams / scratch sets so a chunk's march runs under its predecessor's fused kernel.

The evaluation modes keep everything on the device: rays from ``RayGenerator.RaysOfCamera`` / ``RaysFromPose``
(``f2b_camera_rays``), images rendered back to back by the same tiled loop, and for ``TestImages`` the reference's
quantisation and MSE as device tensor ops with one host sync for all PSNRs.  Image writing is left to the caller.

``TestImages`` also scores every view the way the paper's numbers are computed, by the reference's evaluation script
(scripts/eval.py): 8-bit PSNR and SSIM of the PNGs ``TestImages`` would write, in one kernel per view
(``f2b_image_metrics``, csrc/metrics.cu); ``ImageMetrics`` scores any image pair the same way.  LPIPS is not computed.
"""
import numpy as np
import torch

from ._lib import call, stream
from .sampler import VALIDATE

RAY_BATCH_SIZE = 8192          # ExpRunner.cpp:268
_METRICS_WORK_BYTES = 16 * 1024   # F2B_METRICS_WORK_BYTES (include/f2nerf_b200.h)


def _to_dev(x, dev):
    x = x.to(torch.float32)
    if x.is_cuda:
        return x.contiguous()
    return (x.contiguous().pin_memory() if torch.cuda.is_available() else x).to(dev, non_blocking=True)


def _render_rays(renderer, o, d, ray_batch_size, dev):
    """The tiled VALIDATE-mode render of one image's rays (device [N,3] each) -> device (colors [N,3], first_oct_disp [N,1],
    pred_disp [N,1]), normalised as ExpRunner.cpp:289-290.  No host sync on the fused path.  The caller sets VALIDATE mode."""
    n_rays = d.shape[0]
    colors = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
    first = torch.full((n_rays, 1), 1., dtype=torch.float32, device=dev)
    disp = torch.zeros((n_rays, 1), dtype=torch.float32, device=dev)
    if renderer._fused_forward_ok(n_rays):
        # Tiled renderer: every chunk is march + ONE fused kernel (Renderer.render_forward) that writes its rows of the
        # device-resident image directly; no host sync, no per-chunk copies.  Two chunks are in flight on two streams with
        # two march scratch sets, so chunk k+1's march (per-ray latency bound, ~20 % occupancy) runs under chunk k's
        # fused kernel (gather bound).
        main = torch.cuda.current_stream(dev)
        lanes = [renderer._side_stream(dev, 3), renderer._side_stream(dev, 4)]
        ready = torch.cuda.Event()
        ready.record(main)
        disp_flat, depth = disp.view(-1), torch.empty((n_rays,), dtype=torch.float32, device=dev)
        alive = []
        for k, i in enumerate(range(0, n_rays, ray_batch_size)):
            j = min(i + ray_batch_size, n_rays)
            st = lanes[k % 2]
            if k < 2:
                st.wait_event(ready)
            with torch.cuda.stream(st):
                r = renderer.render_forward(o[i:j], d[i:j], out=(colors[i:j], disp_flat[i:j], depth[i:j]), lane=1 + k % 2)
                first[i:j] = r.first_oct_dis.reshape(-1, 1)
            alive.append(r)                                  # allocations of a lane stay referenced until the join below
        for st in lanes:
            main.wait_stream(st)
        del alive
    else:
        for i in range(0, n_rays, ray_batch_size):
            j = min(i + ray_batch_size, n_rays)
            r = renderer.Render(o[i:j], d[i:j], None, None)
            colors[i:j] = r.colors
            disp[i:j, 0] = r.disparity.reshape(-1)
            if r.first_oct_dis is not None and r.first_oct_dis.numel() == (j - i):
                first[i:j] = r.first_oct_dis.reshape(-1, 1)
    disp = disp / disp.max()                                     # ExpRunner.cpp:289-290
    first = first.min() / first
    return colors, first, disp


class _Validate:
    """VALIDATE mode for the duration of a block, the previous mode restored on every exit (exceptions included)."""

    def __init__(self, renderer):
        self.gdp = renderer.global_data_pool_

    def __enter__(self):
        self.prev = self.gdp.mode_
        self.gdp.mode_ = VALIDATE                                # the reference's callers set it (ExpRunner.cpp:304,325,346)

    def __exit__(self, *exc):
        self.gdp.mode_ = self.prev
        return False


def _device_of(renderer, device):
    return torch.device(device) if device is not None else renderer.app_emb_.device


@torch.no_grad()
def RenderWholeImage(renderer, rays_o, rays_d, bounds=None, ray_batch_size=RAY_BATCH_SIZE, device=None):
    """-> (pred_colors [N,3], first_oct_disp [N,1], pred_disp [N,1]) CPU float32, like the reference.
    ``rays_o`` / ``rays_d``: [N,3] CPU or CUDA tensors; ``bounds`` is accepted and ignored (the sampler marches
    [global_near_, 1e8], PersSampler.cu:322-323)."""
    dev = _device_of(renderer, device)
    with _Validate(renderer):
        colors, first, disp = _render_rays(renderer, _to_dev(rays_o, dev), _to_dev(rays_d, dev), ray_batch_size, dev)
    out = torch.cat([colors, first, disp], 1).cpu()              # the one device->host copy
    return out[:, :3].contiguous(), out[:, 3:4].contiguous(), out[:, 4:5].contiguous()


@torch.no_grad()
def RenderNormals(renderer, rays_o, rays_d, ray_batch_size=RAY_BATCH_SIZE, device=None):
    """-> normals [N,3] CPU float32: the normal map of the rays in the normalised scene frame (DESIGN.md §3j).  Per ray,
    N = sum_i w_i n_i over the samples the VALIDATE render keeps, with n_i = -g_i / |g_i| the outward density normal and w_i the
    render's weights; the result is N / |N|, 0 where N = 0 (rays that miss the scene included).  The rays are rendered in the
    tiled loop of ``RenderWholeImage`` (two streams, ``render_forward`` per chunk), each chunk followed on its stream by the
    normals kernel over the chunk's slots; one device->host copy at the end.  The sums run in a fixed order, so a view gets the
    same bits on every run and for any ``ray_batch_size``.  Turning the map into camera coordinates is one rotation by the
    camera's pose, left to the caller."""
    from . import ops
    dev = _device_of(renderer, device)
    o, d = _to_dev(rays_o, dev), _to_dev(rays_d, dev)
    n_rays = d.shape[0]
    normals = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
    if n_rays == 0:
        return normals.cpu()
    f = renderer.scene_field_
    trans = renderer.pts_sampler_.pers_trans_gpu_
    with _Validate(renderer):
        main = torch.cuda.current_stream(dev)
        lanes = [renderer._side_stream(dev, 3), renderer._side_stream(dev, 4)]
        ready = torch.cuda.Event()
        ready.record(main)
        f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
        unused = [(f32(ray_batch_size, 3), f32(ray_batch_size), f32(ray_batch_size)) for _ in lanes]   # colours etc., per lane
        alive = []
        for k, i in enumerate(range(0, n_rays, ray_batch_size)):
            j = min(i + ray_batch_size, n_rays)
            st = lanes[k % 2]
            if k < 2:
                st.wait_event(ready)
            with torch.cuda.stream(st):
                r = renderer.render_forward(o[i:j], d[i:j], out=tuple(u[:j - i] for u in unused[k % 2]), lane=1 + k % 2)
                ops.render_normals_slots(trans, f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_,
                                         f.mlp_.params_f16(), r._keep[0], r.kept_counts, r._w_slots, out=normals[i:j])
            alive.append(r)                                  # allocations of a lane stay referenced until the join below
        for st in lanes:
            main.wait_stream(st)
        del alive
    return normals.cpu()                                         # the one device->host copy


def quantify(x):
    """ExpRunner::TestImages' ``quantify`` (ExpRunner.cpp:360-362): (x.clip(0,1) * 255).to(uint8).to(float32) / 255, bit-exact
    on the device.  The reference runs it on CPU tensors, where dividing by the scalar 255 is a true division; ATen's CUDA
    kernel would multiply by the rounded reciprocal instead (126 of the 256 levels then differ by one ulp), so the divisor is
    a device tensor here, which keeps the division."""
    return (x.clip(0., 1.) * 255.).to(torch.uint8).to(torch.float32) / torch.full((), 255., dtype=torch.float32, device=x.device)


def ssim_taps(filter_size=11, filter_sigma=1.5):
    """rgb_ssim's 1D Gaussian blur filter (scripts/eval.py:41-45) by the same float64 numpy expression, so that the device never
    evaluates ``exp`` for it: exp(-0.5 ((k - hw + shift) / sigma)^2) for k < filter_size, divided by its numpy sum."""
    hw = filter_size // 2
    shift = (2 * hw - filter_size + 1) / 2
    filt = np.exp(-0.5 * ((np.arange(filter_size) - hw + shift) / filter_sigma) ** 2)
    return filt / np.sum(filt)


SSIM_TAPS = ssim_taps()        # host memory; f2b_image_metrics reads it during each call


def psnr_8bit(sse, n_values):
    """skimage's peak_signal_noise_ratio on two uint8 images (scripts/eval.py:98): data range 255 (the dtype's), MSE the float64
    mean of the squared differences, 10 log10(255^2 / MSE); ``inf`` for equal images, as skimage gives.  ``sse`` is the exact
    integer sum, so the MSE is the one numpy forms."""
    if sse == 0:
        return float("inf")
    return float(10. * np.log10(65025. / (np.float64(sse) / np.float64(n_values))))


def _image_metrics(pred, gt):
    """f2b_image_metrics on one contiguous [H,W,3] fp32 pair on the current device -> device tensors (sse int64 [1], ssim_sum
    float64 [1]).  No host sync."""
    sse = torch.empty((1,), dtype=torch.int64, device=pred.device)
    ssim_sum = torch.empty((1,), dtype=torch.float64, device=pred.device)
    work = torch.empty((_METRICS_WORK_BYTES,), dtype=torch.uint8, device=pred.device)
    call("f2b_image_metrics", pred, gt, pred.shape[0], pred.shape[1], SSIM_TAPS.ctypes.data, work, sse, ssim_sum, stream())
    return sse, ssim_sum


def _ssim_count(H, W):
    return (H - 10) * (W - 10) * 3                               # the 'valid' convolution's outputs, all channels


@torch.no_grad()
def ImageMetrics(pred, gt):
    """The PSNR and SSIM of the reference's evaluation script (scripts/eval.py:94-100) for one image pair, on the device ->
    {"psnr_8bit": float, "ssim": float}.  ``pred`` and ``gt`` are [H,W,3] CUDA tensors with values in [0,1] and H, W >= 11
    (smaller images raise F2BError).  Both are scored as the 8-bit images the script reads:
    - pred as ``TestImages`` writes it (Utils::WriteImageTensor, ImageIO.cpp:28-32): trunc(clip(x,0,1) * 255).  Raw and
      ``quantify``-ed colours give the same bytes.
    - gt as rint(clip(x,0,1) * 255), the stored byte of an image loaded as u8 / 255.
    PSNR is skimage's peak_signal_noise_ratio (``psnr_8bit``).  SSIM is rgb_ssim(gt / 255., pred / 255., max_val=1) (:29-75) in
    float64: separable 11-tap Gaussian (sigma 1.5, ``ssim_taps``), 'valid' convolution, k1 = 0.01, k2 = 0.03, variances clipped
    at 0, covariance clipped to +-sqrt(var0 var1), mean over the three channels.  LPIPS is not computed."""
    for name, t in (("pred", pred), ("gt", gt)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dim() != 3 or t.shape[2] != 3:
            raise ValueError(f"ImageMetrics: {name} must be a [H,W,3] CUDA tensor")
    if pred.shape != gt.shape or pred.device != gt.device:
        raise ValueError(f"ImageMetrics: pred {tuple(pred.shape)} on {pred.device} and gt {tuple(gt.shape)} on {gt.device} differ")
    H, W = pred.shape[0], pred.shape[1]
    with torch.cuda.device(pred.device):
        sse, ssim_sum = _image_metrics(pred.to(torch.float32).contiguous(), gt.to(torch.float32).contiguous())
        sse, ssim_sum = torch.cat([sse.double(), ssim_sum]).tolist()
    return {"psnr_8bit": psnr_8bit(int(sse), H * W * 3), "ssim": ssim_sum / _ssim_count(H, W)}


@torch.no_grad()
def TestImages(renderer, dataset, ray_batch_size=RAY_BATCH_SIZE, device=None):
    """ExpRunner::TestImages (ExpRunner.cpp:343-391) on ``dataset.test_set_`` ->
    {"psnr": {idx: float}, "mean_psnr": float, "colors": [[H,W,3]], "disparity": [[H,W,1]], "first_oct_dis": [[H,W,1]],
     "psnr_8bit": {idx: float}, "mean_psnr_8bit": float, "ssim": {idx: float}, "mean_ssim": float}
    (device tensors, colours quantised like the reference's PNGs).  The MSE against ``dataset.image_tensors_`` is
    accumulated in float64 on the device and PSNR = 20 log10(1 / sqrt(mse)) (:369).  "psnr_8bit" and "ssim" are what the
    reference's evaluation script reports for the written PNGs (``ImageMetrics``, scripts/eval.py:94-100), computed from the
    quantised colours behind each view's render.  The test images render back to back and all values come to the host in one
    copy at the end."""
    dev = _device_of(renderer, device)
    H, W = dataset.height_, dataset.width_
    out = {"colors": [], "disparity": [], "first_oct_dis": []}
    psnrs, scores = [], []
    with _Validate(renderer):
        for idx in dataset.test_set_:
            rays_o, rays_d, _ = dataset.RaysOfCamera(idx)
            colors, first, disp = _render_rays(renderer, rays_o, rays_d, ray_batch_size, dev)
            q = quantify(colors.reshape(H, W, 3))
            gt = dataset.image_tensors_[idx].reshape(H, W, 3)
            mse = (q.double() - gt.double()).square().mean()
            psnrs.append(20. * torch.log10(1. / torch.sqrt(mse)))
            sse, ssim_sum = _image_metrics(q, gt.contiguous())
            scores.append(torch.cat([sse.double(), ssim_sum]))          # SSE < 2^53: exact in float64
            out["colors"].append(q)
            out["disparity"].append(disp.reshape(H, W, 1))
            out["first_oct_dis"].append(first.reshape(H, W, 1))
    rows = torch.cat([torch.stack(psnrs)[:, None], torch.stack(scores)], 1).tolist() if psnrs else []   # the one host sync
    vals = [r[0] for r in rows]
    out["psnr"] = {int(i): float(v) for i, v in zip(dataset.test_set_, vals)}
    out["mean_psnr"] = sum(vals) / len(vals) if vals else float("nan")
    out["psnr_8bit"] = {int(i): psnr_8bit(int(r[1]), H * W * 3) for i, r in zip(dataset.test_set_, rows)}
    out["ssim"] = {int(i): r[2] / _ssim_count(H, W) for i, r in zip(dataset.test_set_, rows)}
    for k in ("psnr_8bit", "ssim"):
        out["mean_" + k] = sum(out[k].values()) / len(rows) if rows else float("nan")
    return out


@torch.no_grad()
def RenderPath(renderer, dataset, reso_level=1, ray_batch_size=RAY_BATCH_SIZE, device=None):
    """ExpRunner::RenderPath (ExpRunner.cpp:322-341) over ``dataset.render_poses_`` -> list of device tuples
    (colors [h,w,3], first_oct_dis [h,w,1], disparity [h,w,1]) with h, w = height // reso_level, width // reso_level."""
    if dataset.render_poses_ is None:
        raise ValueError("RenderPath: the dataset has no render_poses")
    dev = _device_of(renderer, device)
    h, w = dataset.height_ // int(reso_level), dataset.width_ // int(reso_level)
    frames = []
    with _Validate(renderer):
        for pose in dataset.render_poses_:
            rays_o, rays_d, _ = dataset.RaysFromPose(pose, reso_level)
            colors, first, disp = _render_rays(renderer, rays_o, rays_d, ray_batch_size, dev)
            frames.append((colors.reshape(h, w, 3), first.reshape(h, w, 1), disp.reshape(h, w, 1)))
    return frames


@torch.no_grad()
def RenderAllImages(renderer, dataset, ray_batch_size=RAY_BATCH_SIZE, device=None):
    """ExpRunner::RenderAllImages / VisualizeImage (ExpRunner.cpp:295-320): for every camera the device image
    cat([GT | pred | first_oct_dis x3 | disparity x3], width) [H, 4W, 3] (GT zeros when the dataset holds no images)."""
    dev = _device_of(renderer, device)
    H, W = dataset.height_, dataset.width_
    images = []
    with _Validate(renderer):
        for idx in range(dataset.n_images_):
            rays_o, rays_d, _ = dataset.RaysOfCamera(idx)
            colors, first, disp = _render_rays(renderer, rays_o, rays_d, ray_batch_size, dev)
            gt = (dataset.image_tensors_[idx].reshape(H, W, 3) if dataset.image_tensors_ is not None
                  else torch.zeros((H, W, 3), dtype=torch.float32, device=dev))
            images.append(torch.cat([gt, colors.reshape(H, W, 3), first.reshape(H, W, 1).expand(H, W, 3),
                                     disp.reshape(H, W, 1).expand(H, W, 3)], 1))
    return images
