"""ctypes binding of oracle/libcamrays_oracle.so (oracle/camera_rays.c: the CPU restatement of the reference's whole-camera
rays) for the tests.  Test infrastructure: never imported by the f2nerf_b200 package."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "oracle", "camera_rays.c")
SO = os.path.join(ROOT, "oracle", "libcamrays_oracle.so")


def build():
    """The library build() made; (re)compiled when missing or older than its source — into a temporary directory when the
    tree is read-only."""
    if os.path.exists(SO) and os.path.getmtime(SO) >= os.path.getmtime(SRC):
        return SO
    out = SO if os.access(os.path.dirname(SO), os.W_OK) else os.path.join(tempfile.mkdtemp(prefix="f2b_camrays_"), "libcamrays_oracle.so")
    subprocess.check_call(["gcc", "-O2", "-march=x86-64-v3", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                           "-shared", "-fPIC", SRC, "-o", out, "-lm"])
    return out


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def camera_rays(pose, intri, dist_params, height, width, out_h, out_w, idx=None):
    """Dataset::RaysOfCamera / RaysFromPose restated (orc_camera_rays) for one camera -> (rays_o, rays_d) [n,3] for the ray
    indices ``idx`` (a*out_w + b), or for all out_h*out_w rays when idx is None."""
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    idx = None if idx is None else np.ascontiguousarray(idx, dtype=np.int32)
    n = out_h * out_w if idx is None else idx.shape[0]
    rays_o, rays_d = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
    I = ctypes.c_int
    lib().orc_camera_rays(_p(f(pose)), _p(f(intri)), _p(f(dist_params)), I(height), I(width), I(out_h), I(out_w), _p(idx), I(n),
                          _p(rays_o), _p(rays_d))
    return rays_o, rays_d
