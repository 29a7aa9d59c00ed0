"""ctypes binding of tests/locate_oracle.c (the CPU restatement of f2b_locate_points).  Test infrastructure: never imported by
the f2nerf_b200 package.  The library is compiled on first use into a temporary directory, so the tree may be read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "locate_oracle.c")
ORACLE_SRC = os.path.join(os.path.dirname(HERE), "oracle", "f2_oracle.c")

_lib = None


def build():
    """-> path of the compiled library, rebuilt whenever either source changes."""
    h = hashlib.sha256()
    for p in (SRC, ORACLE_SRC):
        with open(p, "rb") as f:
            h.update(f.read())
    out_dir = os.path.join(tempfile.gettempdir(), f"f2b_locate_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"liblocate_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call(["gcc", "-O2", "-march=x86-64-v3", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-shared",
                               "-fPIC", SRC, "-o", tmp, "-lm"])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def locate_points(tree_nodes, trans, pts):
    """orc_locate_points -> (warped [n,3] f32, anchors [n,2] i32 = (trans_idx, leaf node))."""
    nodes = np.ascontiguousarray(tree_nodes, np.uint8)
    trans = np.ascontiguousarray(trans, np.uint8)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n = pts.shape[0]
    warped, anchors = np.zeros((n, 3), np.float32), np.zeros((n, 2), np.int32)
    lib().orc_locate_points(_p(nodes), _p(trans), _p(pts), ctypes.c_int(n), _p(warped), _p(anchors))
    return warped, anchors
