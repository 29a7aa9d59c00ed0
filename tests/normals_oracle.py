"""ctypes binding of tests/normals_oracle.c (the CPU restatement of the gradient kernel's warp Jacobian) and a float64 twin of
the pieces of the density gradient.  Test infrastructure: never imported by the f2nerf_b200 package.  The library is compiled
on first use into a temporary directory, so the tree may be read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "normals_oracle.c"), os.path.join(HERE, "locate_oracle.c"),
        os.path.join(os.path.dirname(HERE), "oracle", "f2_oracle.c")]
F64 = torch.float64

_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in SRCS:
            with open(p, "rb") as f:
                h.update(f.read())
        out_dir = os.path.join(tempfile.gettempdir(), f"f2b_normals_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libnormals_oracle_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-march=x86-64-v3", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-shared",
                                   "-fPIC", SRCS[0], "-o", tmp, "-lm"])
            os.replace(tmp, so)
        _lib = ctypes.CDLL(so)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def warp_jacobian(tree_nodes, trans, pts):
    """orc_warp_jacobian -> J [n,3,3] float32."""
    nodes = np.ascontiguousarray(tree_nodes, np.uint8)
    trans = np.ascontiguousarray(trans, np.uint8)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    jac = np.zeros((pts.shape[0], 3, 3), np.float32)
    lib().orc_warp_jacobian(_p(nodes), _p(trans), _p(pts), ctypes.c_int(pts.shape[0]), _p(jac))
    return jac


# ------------------------------------------------------------------------------------------------------------ float64 twin
def trans_arrays(trans_u8):
    """TransInfo blobs -> (w2xz [T,12,2,4], weight [T,3,12]) float64."""
    f = np.ascontiguousarray(trans_u8, np.uint8).view(np.float32).reshape(-1, 136).astype(np.float64)
    return f[:, :96].reshape(-1, 12, 2, 4), f[:, 96:132].reshape(-1, 3, 12)


def warp64(w2xz, weight, x):
    """QueryFrameTransform in float64: x [n,3] with per-point w2xz [n,12,2,4], weight [n,3,12] -> [n,3]."""
    xh = np.concatenate([x, np.ones((x.shape[0], 1))], 1)
    xz = np.einsum("nkij,nj->nki", w2xz, xh)
    return np.einsum("nrk,nk->nr", weight, xz[:, :, 0] / xz[:, :, 1])


def jacobian64(w2xz, weight, x, magnitude=False):
    """d warp / d x in float64 -> J [n,3,3] (and, with ``magnitude``, sum_k |weight_rk| |dv_k/dx_c|)."""
    xh = np.concatenate([x, np.ones((x.shape[0], 1))], 1)
    xz = np.einsum("nkij,nj->nki", w2xz, xh)
    a, b = w2xz[:, :, 0, :3], w2xz[:, :, 1, :3]
    dv = (a * xz[:, :, 1:2] - xz[:, :, 0:1] * b) / xz[:, :, 1:2] ** 2            # [n,12,3]
    J = np.einsum("nrk,nkc->nrc", weight, dv)
    if magnitude:
        return J, np.einsum("nrk,nkc->nrc", np.abs(weight), np.abs(dv))
    return J


def corner_weights(frac):
    """Trilinear weights [n,8] of fractions [n,3] (float64, differentiable), corner order 000, 001, ..., 111 (x, y, z bits)."""
    ws = []
    for c in range(8):
        bx, by, bz = (c >> 2) & 1, (c >> 1) & 1, c & 1
        ws.append((frac[:, 0] if bx else 1. - frac[:, 0]) * (frac[:, 1] if by else 1. - frac[:, 1]) *
                  (frac[:, 2] if bz else 1. - frac[:, 2]))
    return torch.stack(ws, 1)


def blend_grad(table, rows, frac, dfeat, magnitude=False):
    """d/dfrac of sum_c w_c(frac) (dfeat . table[rows_c]) by autograd (float64) -> [n,3]; ``magnitude``: the same sum with every
    factor replaced by its absolute value and each dw_c/dfrac by its magnitude (the scale the run's fp32 sums are formed at)."""
    fr = frac.detach().clone().requires_grad_(True)
    s = (table[rows] * dfeat[:, None, :]).sum(-1)                                # [n,8]
    g, = torch.autograd.grad((corner_weights(fr) * s).sum(), fr)
    if not magnitude:
        return g
    sa = (table[rows].abs() * dfeat.abs()[:, None, :]).sum(-1)
    out = []
    for a in range(3):
        m = torch.zeros_like(fr[:, 0])
        for c in range(8):
            w = torch.ones_like(m)
            for k in range(3):
                if k != a:
                    bit = (c >> (2 - k)) & 1
                    w = w * (frac[:, k] if bit else 1. - frac[:, k])
            m = m + w * sa[:, c]
        out.append(m)
    return g, torch.stack(out, 1)
