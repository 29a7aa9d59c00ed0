"""RayGenerator — SURVEY §8(f) N3: ``Dataset::RandRaysData`` / ``Img2WorldRayFlex`` (src/Dataset/Dataset.cpp:275-298,
src/Dataset/Dataset.cu:100-152), the step immediately before the path.

The reference draws camera / row / column indices on the CPU generator, gathers the ground-truth colours from a CPU
image tensor (50 x 540 x 960 x 3 fp32), copies three tensors host->device and launches the ray kernel.  Here the camera
tables AND the images live in HBM; the index draws stay the same ``torch.randint`` calls on the same (CPU) generator in
the same order — so a shared ``torch.manual_seed`` reproduces the reference's batch — and everything after the draws
is two small kernels behind the C ABI (``f2b_img2world_rays``, ``f2b_gather_pixels``): one 48 KB host->device copy per
batch instead of three plus a CPU gather.  The whole-camera rays of the evaluation modes (``RaysOfCamera`` /
``RaysFromPose``, Dataset.cpp:177-218) are one more kernel, ``f2b_camera_rays``.

``load_dataset`` reads a reference data directory the way ``Dataset::Dataset`` and ``NormalizeScene`` do (Dataset.cpp:16-146):
camera tables, scene normalisation, relaxed bounds, the train/test/val split and the images.  The normalisation is the
reference's own ATen ops on the device in the same order, so the camera tables — and with them every ray — are bit-identical
to the reference program's on the GPU.  Images are decoded with PIL (libjpeg), the reference with stb_image: JPEG pixels can
differ by a level or two (on ngp_fox, 55 of 1536 sampled channel values, at most 2/255).  The reference's evaluation script
reads ground truth through libjpeg as well.  PNG images decode identically.
"""
import os

import numpy as np
import torch

from ._lib import call, stream

DATA_TRAIN_SET, DATA_TEST_SET, DATA_VAL_SET = 1, 2, 4           # Dataset.h
_IMAGE_SUFFIXES = ("*.jpg", "*.png", "*.JPG", "*.jpeg")         # scripts/run.py:21


class RayGenerator:
    def __init__(self, poses, intri, dist_params, bounds, images=None, height=None, width=None, train_set=None, val_set=(),
                 test_set=(), device="cuda", render_poses=None):
        """poses [n,3,4], intri [n,3,3], dist_params [n,4], bounds [n,2] (float32, as ``Dataset`` holds them);
        images [n,H,W,3] float32 in [0,1] or None (then pass height/width and no colours are returned);
        render_poses [m,3,4] or None: the novel-view path ``RenderPath`` follows, normalised like ``Dataset::render_poses_``
        (Dataset.cpp:58-70)."""
        dev = torch.device(device)
        f = lambda t: torch.as_tensor(t, dtype=torch.float32).to(dev).contiguous()
        self.poses_, self.intri_, self.dist_params_, self.bounds_ = f(poses), f(intri), f(dist_params), f(bounds)
        self.render_poses_ = None if render_poses is None else f(render_poses).reshape(-1, 3, 4)
        self.n_images_ = self.poses_.shape[0]
        self.image_tensors_ = None if images is None else f(images)
        self.height_ = int(height if images is None else self.image_tensors_.shape[1])
        self.width_ = int(width if images is None else self.image_tensors_.shape[2])
        self.train_set_ = list(range(self.n_images_)) if train_set is None else [int(i) for i in train_set]
        self.val_set_, self.test_set_ = [int(i) for i in val_set], [int(i) for i in test_set]

    def Img2WorldRayFlex(self, cam_indices, ij):
        """Dataset::Img2WorldRayFlex: cam_indices [n] i32, ij [n,2] i32 (row, col) on the device -> (rays_o, rays_d)."""
        n = cam_indices.shape[0]
        dev = self.poses_.device
        rays_o = torch.empty((n, 3), dtype=torch.float32, device=dev)
        rays_d = torch.empty((n, 3), dtype=torch.float32, device=dev)
        call("f2b_img2world_rays", self.poses_, self.intri_, self.dist_params_, cam_indices, ij, n, rays_o, rays_d, stream())
        return rays_o, rays_d

    def RandRaysData(self, batch_size, sets=DATA_TRAIN_SET):
        """Dataset::RandRaysData -> ((rays_o, rays_d, bounds), gt_colors | None, cam_indices i32).  Same CPU draws, in
        the same order, as the reference (Dataset.cpp:287-290)."""
        img_idx = []
        if sets & DATA_TRAIN_SET:
            img_idx += self.train_set_
        if sets & DATA_VAL_SET:
            img_idx += self.val_set_
        if sets & DATA_TEST_SET:
            img_idx += self.test_set_
        cur_set = torch.tensor(img_idx, dtype=torch.int32)
        cam = cur_set[torch.randint(len(img_idx), (batch_size,), dtype=torch.int64)]
        i = torch.randint(0, self.height_, (batch_size,), dtype=torch.int64)
        j = torch.randint(0, self.width_, (batch_size,), dtype=torch.int64)
        packed = torch.stack([cam.to(torch.int32), i.to(torch.int32), j.to(torch.int32)], 1)     # one H2D copy [n,3] i32
        packed = (packed.pin_memory() if torch.cuda.is_available() else packed).to(self.poses_.device, non_blocking=True)
        cam_d, ij_d = packed[:, 0].contiguous(), packed[:, 1:3].contiguous()
        rays_o, rays_d = self.Img2WorldRayFlex(cam_d, ij_d)
        gt = None
        if self.image_tensors_ is not None:
            gt = torch.empty((batch_size, 3), dtype=torch.float32, device=self.poses_.device)
            call("f2b_gather_pixels", self.image_tensors_, cam_d, ij_d, self.height_, self.width_, batch_size, gt, stream())
        bounds = self.bounds_[cam_d.long()].contiguous()
        return (rays_o, rays_d, bounds), gt, cam_d

    def _camera_rays(self, pose, intri, dist_params, out_h, out_w):
        n = out_h * out_w
        dev = self.poses_.device
        rays_o = torch.empty((n, 3), dtype=torch.float32, device=dev)
        rays_d = torch.empty((n, 3), dtype=torch.float32, device=dev)
        call("f2b_camera_rays", pose, intri, dist_params, self.height_, self.width_, out_h, out_w, rays_o, rays_d, stream())
        return rays_o, rays_d

    def RaysOfCamera(self, idx, reso_level=1):
        """Dataset::RaysOfCamera (Dataset.cpp:177-196) -> (rays_o, rays_d, bounds) [H*W,3|3|2] on the device, ray a*W + b
        through pixel (a, b).  ``reso_level`` is ignored, as in the reference."""
        idx = int(idx)
        rays_o, rays_d = self._camera_rays(self.poses_[idx], self.intri_[idx], self.dist_params_[idx], self.height_, self.width_)
        bounds = self.bounds_[idx].expand(rays_o.shape[0], 2).contiguous()
        return rays_o, rays_d, bounds

    def RaysFromPose(self, pose, reso_level=1):
        """Dataset::RaysFromPose (Dataset.cpp:198-218): the (height // reso_level) x (width // reso_level) grid spread over
        the full image, camera 0's intrinsics and distortion, the near / far bounds of all cameras (device reductions,
        no host sync) -> (rays_o, rays_d, bounds) on the device."""
        out_h, out_w = self.height_ // int(reso_level), self.width_ // int(reso_level)
        pose = torch.as_tensor(pose, dtype=torch.float32).to(self.poses_.device).reshape(3, 4).contiguous()
        rays_o, rays_d = self._camera_rays(pose, self.intri_[0], self.dist_params_[0], out_h, out_w)
        near_far = torch.stack([self.bounds_[:, 0].min(), self.bounds_[:, 1].max()])
        return rays_o, rays_d, near_far.expand(rays_o.shape[0], 2).contiguous()


def _npy_f32(path, dev):
    """A float64 .npy table cast to float32 on the host, then moved (Dataset.cpp:37-38)."""
    return torch.from_numpy(np.load(path).astype(np.float64)).to(torch.float32).to(dev)


def image_paths(data_path, factor, n_images):
    """The image files of a data directory, in camera order: the first ``n_images`` lines of ``image_list.txt``
    (Dataset.cpp:78-86), else the listing scripts/run.py:18-35 would write (images_{round(factor)}/*.{jpg,png,JPG,jpeg},
    or images/ and images_1/ at factor 1, sorted).  A listed path is looked up against the working directory first, which is
    how the reference program resolves it, then against the data directory."""
    list_file = os.path.join(data_path, "image_list.txt")
    if os.path.isfile(list_file):
        with open(list_file) as f:
            lines = [ln.rstrip("\r\n") for ln in f][:n_images]
        paths = []
        for ln in lines:
            cands = [ln] if os.path.isabs(ln) else [ln, os.path.join(data_path, ln)]
            hit = next((c for c in cands if os.path.isfile(c)), None)
            if hit is None:
                raise FileNotFoundError(f"load_dataset: {list_file} lists {ln!r}, found neither in the working directory "
                                        f"nor in {data_path}")
            paths.append(hit)
    else:
        import glob
        subdirs = ("images", "images_1") if 0.999 < factor < 1.001 else (f"images_{int(np.round(factor))}",)
        paths = sorted(p for suf in _IMAGE_SUFFIXES for d in subdirs for p in glob.glob(os.path.join(data_path, d, suf)))
    if len(paths) != n_images:
        raise ValueError(f"load_dataset: {n_images} cameras in {data_path}/cams_meta.npy but {len(paths)} images")
    return paths


def read_image_u8(path):
    """One image file -> uint8 [H,W,3] (PIL)."""
    from PIL import Image
    with Image.open(path) as im:
        if im.mode in ("RGBA", "LA", "PA") or "transparency" in im.info:
            raise ValueError(f"load_dataset: {path} has an alpha channel; the renderer scores RGB images")
        return np.asarray(im.convert("RGB"))


def load_dataset(data_path, factor, bounds_factor, device="cuda"):
    """``Dataset::Dataset`` + ``NormalizeScene`` (Dataset.cpp:16-146) for a reference data directory -> ``RayGenerator``.

    - ``cams_meta.npy`` float64 [n,27] (pose 12, intrinsics 9, distortion 4, bounds 2), cast to float32 on the host;
      intrinsics rows 0-1 divided by ``factor``.
    - Scene normalisation on the device: center = mean camera position, radius = the largest distance from it; positions,
      bounds and the ``poses_render.npy`` path (when present) moved and scaled by it.  Same ATen ops in the same order as the
      reference (a division by a Python float is a multiply by its float reciprocal on CUDA), so on a CUDA device the
      tables are bit-identical to the reference program's.
    - Bounds scaled by ``bounds_factor`` = (near, far), then clamped to [1e-2, 1e9].
    - Train / test / val split from the bits of ``split.npy``, else every 8th camera is a test camera.
    - Images (``image_paths``) decoded to uint8 on the host, uploaded, and divided by 255 on the device as a true
      division (the reference divides on the CPU; see ``eval.quantify``).

    The result also carries ``center_`` (device [3]) and ``radius_`` (float) of the normalisation."""
    dev = torch.device(device)
    factor = float(np.float32(factor))                           # config["factor"].as<float>()
    bf = [float(np.float32(v)) for v in bounds_factor]           # config["bounds_factor"].as<std::vector<float>>()
    meta = os.path.join(data_path, "cams_meta.npy")
    if not os.path.isfile(meta):
        raise FileNotFoundError(f"load_dataset: {meta} does not exist")
    cam_data = _npy_f32(meta, dev)
    n_images = cam_data.shape[0]
    cam_data = cam_data.reshape(n_images, 27)
    poses = cam_data[:, 0:12].reshape(-1, 3, 4).contiguous()
    intri = cam_data[:, 12:21].reshape(-1, 3, 3).contiguous()
    intri[:, 0:2, 0:3] = intri[:, 0:2, 0:3] / factor
    dist_params = cam_data[:, 21:25].reshape(-1, 4).contiguous()
    bounds = cam_data[:, 25:27].reshape(-1, 2).contiguous()

    # NormalizeScene (Dataset.cpp:124-143)
    cam_pos = poses[:, 0:3, 3].clone()
    center = cam_pos.mean(0)
    bias = cam_pos - center.unsqueeze(0)
    radius = float(torch.linalg.norm(bias, 2, -1, False).max().item())
    cam_pos = (cam_pos - center.unsqueeze(0)) / radius
    poses[:, 0:3, 3] = cam_pos
    poses = poses.contiguous()
    bounds = (bounds / radius).contiguous()

    render_poses = None
    render_file = os.path.join(data_path, "poses_render.npy")
    if os.path.isfile(render_file):                              # Dataset.cpp:58-70
        render_poses = _npy_f32(render_file, dev).reshape(-1, 3, 4)
        render_poses[:, 0:3, 3] = (render_poses[:, 0:3, 3] - center.unsqueeze(0)) / radius

    bounds = torch.stack([bounds[..., 0] * bf[0], bounds[..., 1] * bf[1]], -1).contiguous()     # Dataset.cpp:73-76
    bounds.clamp_(1e-2, 1e9)

    split_file = os.path.join(data_path, "split.npy")
    train_set, test_set, val_set = [], [], []
    if os.path.isfile(split_file):                               # Dataset.cpp:89-100
        split = np.load(split_file).reshape(-1).astype(np.uint8)
        if split.shape[0] != n_images:
            raise ValueError(f"load_dataset: {split_file} has {split.shape[0]} entries for {n_images} cameras")
        for i, st in enumerate(int(s) for s in split):
            if st & 1:
                train_set.append(i)
            if st & 2:
                test_set.append(i)
            if st & 4:
                val_set.append(i)
    else:                                                        # Dataset.cpp:101-106
        for i in range(n_images):
            (test_set if i % 8 == 0 else train_set).append(i)

    u8 = np.stack([read_image_u8(p) for p in image_paths(data_path, factor, n_images)])
    images = torch.from_numpy(u8).to(dev).to(torch.float32) / torch.full((), 255., dtype=torch.float32, device=dev)

    ds = RayGenerator(poses, intri, dist_params, bounds, images=images, train_set=train_set, val_set=val_set,
                      test_set=test_set, device=dev, render_poses=render_poses)
    ds.center_, ds.radius_ = center, radius
    return ds
