"""RayGenerator — SURVEY §8(f) N3: ``Dataset::RandRaysData`` / ``Img2WorldRayFlex`` (src/Dataset/Dataset.cpp:275-298,
src/Dataset/Dataset.cu:100-152), the step immediately before the path.

The reference draws camera / row / column indices on the CPU generator, gathers the ground-truth colours from a CPU
image tensor (50 x 540 x 960 x 3 fp32), copies three tensors host->device and launches the ray kernel.  Here the camera
tables AND the images live in HBM; the index draws stay the same ``torch.randint`` calls on the same (CPU) generator in
the same order — so a shared ``torch.manual_seed`` reproduces the reference's batch — and everything after the draws
is two small kernels behind the C ABI (``f2b_img2world_rays``, ``f2b_gather_pixels``): one 48 KB host->device copy per
batch instead of three plus a CPU gather.  The whole-camera rays of the evaluation modes (``RaysOfCamera`` /
``RaysFromPose``, Dataset.cpp:177-218) are one more kernel, ``f2b_camera_rays``.  Image loading, pose normalisation and the train/test split
(``Dataset::Dataset``, Dataset.cpp:16-190) are out of scope: the tensors are handed in.
"""
import torch

from ._lib import call, stream

DATA_TRAIN_SET, DATA_TEST_SET, DATA_VAL_SET = 1, 2, 4           # Dataset.h


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
