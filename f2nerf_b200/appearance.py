"""Appearance of a trained scene (DESIGN.md §3m): fit the per-image appearance row to a photo, and score held-out views the way
NeRF-in-the-wild methods are scored.

The shader adds a 16-float row to its input, [1, feat 1..15] + row; training learns one row per training image
(``Renderer.app_emb_``).  ``Renderer.appearance_row`` turns an ``appearance=`` argument into a row, and the evaluation and geometry
functions render with it through ``f2b_render_fwd_fused_app``.

``FitAppearance`` fits a row to a photo with the scene held fixed: per iteration the VALIDATE render of ``n_rays`` seeded pixels
through the launch sequences with the row in phase 2's embedding path (``pose._render``), the mean squared colour error, and its
gradient with respect to the row: the composite and shader-MLP backward to the shader's input rows (``pose._shader_input_bwd``),
summed over the kept samples in a fixed order.  The row is the same for every sample, so that sum is the whole gradient; no field
backward runs.  Nothing of the scene is written: no octree votes, no statistics, no draw from the default CUDA generator, and
``Renderer.sample_result_`` is left alone.

``TestAppearance`` fits each test view's row on the left half of its photo and scores the right half.
"""
import numpy as np
import torch

from . import pose as _pose
from .eval import RAY_BATCH_SIZE, _image_metrics, _render_rays, _ssim_count, _Validate, psnr_8bit, quantify


def left_half_mask(height, width):
    """[H,W] bool: the pixels ``FitAppearance`` fits on in ``TestAppearance``, the columns < W // 2."""
    m = torch.zeros((int(height), int(width)), dtype=torch.bool)
    m[:, :int(width) // 2] = True
    return m


def right_half_pixels(height, width):
    """int64 [H * (W - W // 2)]: the scored pixels a * W + b with b >= W // 2, in row-major order of the [H, W - W // 2] crop."""
    H, W = int(height), int(width)
    return (torch.arange(H)[:, None] * W + torch.arange(W // 2, W)[None, :]).reshape(-1)


def _row_grad(b, d_colors, shader_scale):
    """dL/drow [16] float32 of one rendered batch: sum over the kept samples of dL/d(shader input channels 0..15), un-scaled.  The
    sum runs in float64 in a fixed order (no atomics), so a fit gets the same bits on every run."""
    dev = b.rays_o.device
    if b.n_all <= 0:
        return torch.zeros((16,), dtype=torch.float32, device=dev)
    _, _, d_in16 = _pose._shader_input_bwd(b, d_colors, shader_scale)
    return (d_in16[:, :16].double().sum(0) / shader_scale).float()


def _pixels(mask, H, W):
    if mask is None:
        return None
    m = torch.as_tensor(mask)
    if m.shape != (H, W) or m.dtype != torch.bool:
        raise ValueError(f"FitAppearance: mask must be a [{H}, {W}] bool tensor, got {tuple(m.shape)} {m.dtype}")
    cand = torch.nonzero(m.cpu().reshape(-1)).squeeze(1)
    if cand.numel() == 0:
        raise ValueError("FitAppearance: the mask selects no pixel")
    return cand


def FitAppearance(renderer, image, camera, pose, mask=None, init=None, iters=300, n_rays=4096, lr=1e-2, seed=0, dataset=None):
    """Fit the appearance row of the photo ``image`` [H,W,3] (values in [0,1]) taken by ``camera`` at ``pose`` ([3,4] camera to
    world, normalised scene frame; ``camera`` is (intrinsics [3,3], distortion [4]) or a dataset camera's index, as in
    ``RefinePose``).  ``mask``: optional [H,W] bool of the pixels to fit.  ``init``: the starting row (anything
    ``Renderer.appearance_row`` takes; default zeros, the reference's VALIDATE rendering).  Per iteration ``n_rays`` pixels are drawn
    from a ``torch.Generator`` seeded with ``seed`` and Adam (``lr``) steps the row on their mean squared colour error.  The
    defaults have not been tuned.  -> (row [16] float32 on the renderer's device, per-iteration losses list)."""
    if iters < 0 or n_rays <= 0:
        raise ValueError(f"FitAppearance: iters >= 0 and n_rays > 0 required, got {iters}, {n_rays}")
    row0 = renderer.appearance_row(torch.zeros(16) if init is None else init)
    img = torch.as_tensor(image)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"FitAppearance: image must be [H,W,3], got {tuple(img.shape)}")
    H, W = int(img.shape[0]), int(img.shape[1])
    p = _pose._check_pose(pose, "FitAppearance")
    intri, dist = _pose._camera(camera, dataset, H, W, "FitAppearance")
    cand = _pixels(mask, H, W)
    dev = renderer.app_emb_.device
    gt = img.to(device=dev, dtype=torch.float32).reshape(-1, 3)
    o_all, d_all = _pose.rays_from_pose(p, _pose.camera_directions(intri, dist, H, W, dev))
    d_all = _pose._unit(d_all)
    gen = torch.Generator(device="cpu").manual_seed(int(seed))
    row = row0.clone().requires_grad_(True)
    opt = torch.optim.Adam([row], lr=lr)
    losses = []
    for _ in range(int(iters)):
        k = torch.randint(H * W if cand is None else cand.numel(), (int(n_rays),), generator=gen)
        pix = (k if cand is None else cand[k]).to(dev)
        with torch.no_grad():
            b = _pose._render(renderer, o_all[pix].contiguous(), d_all[pix].contiguous(), app=row.detach())
            diff = b.colors - gt[pix]
            loss = diff.square().mean()
            d_colors = diff * (2. / diff.numel())
            g, _, _ = _pose.backed_off(lambda sh, fs: _row_grad(b, d_colors, sh), lambda g: bool(torch.isfinite(g).all()),
                                       "FitAppearance: non-finite appearance gradient")
        row.grad = g
        opt.step()
        losses.append(float(loss))
    return row.detach().clone(), losses


@torch.no_grad()
def _score_right_half(renderer, o, d, gt_crop, app, dev):
    """The right-half crop rendered with ``app`` -> device [3]: the reference's quantised PSNR (as ``TestImages``), the 8-bit SSE and
    the SSIM sum (``ImageMetrics``)."""
    h, w = gt_crop.shape[0], gt_crop.shape[1]
    with _Validate(renderer):
        colors, _, _ = _render_rays(renderer, o, d, RAY_BATCH_SIZE, dev, app)
    q = quantify(colors.reshape(h, w, 3))
    mse = (q.double() - gt_crop.double()).square().mean()
    sse, ssim_sum = _image_metrics(q, gt_crop)
    return torch.cat([(20. * torch.log10(1. / torch.sqrt(mse)))[None], sse.double(), ssim_sum])


def TestAppearance(renderer, dataset, **fit_kwargs):
    """The NeRF-in-the-wild protocol on ``dataset.test_set_``: per view, ``FitAppearance`` on the left half of the photo (columns
    < W // 2, from zeros; ``fit_kwargs`` go to it) and the right half scored with three rows: "none" (no embedding), "mean" (the
    mean of the training views' rows) and "fit".  Only the right half's rays are rendered for the scores.  Metrics on the
    [H, W - W // 2] crop: "psnr" (the reference's quantised PSNR, as ``TestImages``), "psnr_8bit" and "ssim" (as ``ImageMetrics``).
    -> {"none" | "mean" | "fit": {"psnr": {idx: float}, "psnr_8bit": ..., "ssim": ..., "mean_psnr": float, "mean_psnr_8bit": ...,
    "mean_ssim": ...}, "rows": {idx: fitted row [16] CPU}, "mean_row": [16] CPU, "losses": {idx: list}}."""
    if "mask" in fit_kwargs or "init" in fit_kwargs:
        raise ValueError("TestAppearance: the mask and the starting row are the protocol's (left half, zeros)")
    if dataset.image_tensors_ is None:
        raise ValueError("TestAppearance: the dataset holds no images")
    dev = renderer.app_emb_.device
    mean_row = renderer.appearance_row(renderer.app_emb_.detach()[list(dataset.train_set_)].mean(0))
    H, W = dataset.height_, dataset.width_
    left, right = left_half_mask(H, W), right_half_pixels(H, W).to(dev)
    kinds = ("none", "mean", "fit")
    out = {k: {} for k in kinds}
    out.update(rows={}, losses={}, mean_row=mean_row.cpu())
    scores = []
    for idx in dataset.test_set_:
        gt = dataset.image_tensors_[idx].reshape(H, W, 3)
        row, losses = FitAppearance(renderer, gt, idx, dataset.poses_[idx], mask=left, dataset=dataset, **fit_kwargs)
        out["rows"][int(idx)], out["losses"][int(idx)] = row.cpu(), losses
        rays_o, rays_d, _ = dataset.RaysOfCamera(idx)
        o, d = rays_o[right].contiguous(), rays_d[right].contiguous()
        gt_crop = gt[:, W // 2:].contiguous()
        scores.append(torch.stack([_score_right_half(renderer, o, d, gt_crop, app, dev) for app in (None, mean_row, row)]))
    vals = torch.stack(scores).tolist() if scores else []           # [view][kind][psnr, sse, ssim_sum]: one host copy
    n_px = H * (W - W // 2) * 3
    for k, kind in enumerate(kinds):
        rec = out[kind]
        rec["psnr"] = {int(i): v[k][0] for i, v in zip(dataset.test_set_, vals)}
        rec["psnr_8bit"] = {int(i): psnr_8bit(int(v[k][1]), n_px) for i, v in zip(dataset.test_set_, vals)}
        rec["ssim"] = {int(i): v[k][2] / _ssim_count(H, W - W // 2) for i, v in zip(dataset.test_set_, vals)}
        for m in ("psnr", "psnr_8bit", "ssim"):
            rec["mean_" + m] = float(np.mean(list(rec[m].values()))) if vals else float("nan")
    return out
