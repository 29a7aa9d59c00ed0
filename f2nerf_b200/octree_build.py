"""The deterministic half of ``PersOctree``'s constructor (src/PtsSampler/PersSampler.cpp:70-104): the initial octree's
structure and the TV-loss edge pool built over it.

The reference's checkpoint (``PersSampler::States``, PersSampler.cpp:692-701) holds the octree and the warps but not the
edge pool.  On resume the reference keeps the pool its constructor built from the *initial* tree and loads the checkpoint's
nodes and warps underneath it.  That pool depends on the training cameras and the ``pts_sampler`` config alone:

- The initial tree's structure (centres, side lengths, links, ``trans_idx``) is decided by ``GetVisiCams`` (:27-66) and
  ``DistanceSummary`` (:16-25).  Both are deterministic ATen sequences, replayed here op for op, node by node, on the
  device the cameras live on.  On the reference's device (CUDA) the rounding is then the reference's.
- The random draws of ``ConstructTreeNode`` (``rand_pts``, and ``ConstructTrans``' camera picks and PCA) shape only the
  warps' contents.  The checkpoint supplies those, so no draw is replayed and no warp is built here.
- ``trans_idx`` numbers the valid leaves in pre-order, which is the index into the checkpoint's ``pers_trans``.

Building warps, and so training a scene from scratch, is out of scope.  Both functions run once, when a checkpoint is
loaded for training (``checkpoint.load_scene(trainable=True)``); none of this is on the training hot path.
"""
import numpy as np
import torch

from .checkpoint import _libm

N_PROS = 12                          # PersSampler.h:11; a leaf needs N_PROS / 2 visible cameras to hold a warp

TREE_NODE = np.dtype({               # struct alignas(32) TreeNode (PersSampler.h:22-29)
    "names": ["center", "side_len", "parent", "childs", "is_leaf", "trans_idx"],
    "formats": [("<f4", 3), "<f4", "<i4", ("<i4", 8), "u1", "<i4"],
    "offsets": [0, 12, 16, 20, 52, 56],
    "itemsize": 64,
})
EDGE_POOL = np.dtype({               # struct alignas(32) EdgePool (PersSampler.h:31-37)
    "names": ["t_idx_a", "t_idx_b", "center", "dir_0", "dir_1"],
    "formats": ["<i4", "<i4", ("<f4", 3), ("<f4", 3), ("<f4", 3)],
    "offsets": [0, 4, 8, 20, 32],
    "itemsize": 64,
})

f32 = np.float32


def _round_half_away(x):
    """std::round."""
    return np.copysign(np.floor(np.abs(x) + .5), x)


def distance_summary(dis):
    """DistanceSummary (PersSampler.cpp:16-25): the mean log-distance of the nearest quarter of the cameras, exponentiated;
    1e8 without cameras.  Float results and libm's expf, as std::exp on a float calls it."""
    if dis.reshape(-1).shape[0] <= 0:
        return f32(1e8)
    log_dis = torch.log(dis)
    thres = torch.quantile(log_dis, 0.25).item()
    mask = (log_dis < thres).to(torch.float32)
    if f32(mask.sum().item()) < f32(1e-3):
        return f32(_libm.expf(log_dis.mean().item()))
    return f32(_libm.expf(((log_dis * mask).sum() / mask.sum()).item()))


def visible_cams(side_len, center, c2w, intri, bound):
    """GetVisiCams (PersSampler.cpp:27-66): the cameras whose 128-column ray grid hits the cube of side ``side_len`` at
    ``center`` (a [3] tensor) inside the camera's [near, far] bounds.  ``intri`` is the first camera's [3,3] intrinsics,
    as the reference uses for every camera."""
    dev = c2w.device
    half_w, half_h = f32(intri[0, 2].item()), f32(intri[1, 2].item())
    cx, cy, fx, fy = half_w, half_h, f32(intri[0, 0].item()), f32(intri[1, 1].item())
    res_w = 128
    res_h = int(_round_half_away(f32(res_w) / half_w * half_h))
    i = torch.linspace(.5, float(half_h * f32(2.) - f32(.5)), res_h, dtype=torch.float32, device=dev)
    j = torch.linspace(.5, float(half_w * f32(2.) - f32(.5)), res_w, dtype=torch.float32, device=dev)
    i, j = torch.meshgrid(i, j, indexing="ij")
    i, j = i.reshape(-1), j.reshape(-1)
    cam_coords = torch.stack([(j - float(cx)) / float(fx), -(i - float(cy)) / float(fy), -torch.ones_like(j)], -1)
    rays_d = torch.matmul(c2w[:, None, 0:3, 0:3], cam_coords[None, :, :, None])[..., 0]              # [n_cams, n_pix, 3]
    rays_o = c2w[:, None, 0:3, 3].repeat(1, res_h * res_w, 1)
    half = float(f32(side_len) * f32(.5))
    a = ((center - half)[None, None] - rays_o) / rays_d
    b = ((center + half)[None, None] - rays_o) / rays_d
    a = torch.nan_to_num(a, 0., 1e6, -1e6)
    b = torch.nan_to_num(b, 0., 1e6, -1e6)
    aa = torch.maximum(a, b)
    bb = torch.minimum(a, b)
    far = torch.min(aa, -1)[0]
    near = torch.max(bb, -1)[0]
    far = torch.minimum(far, bound[:, None, 1])
    near = torch.maximum(near, bound[:, None, 0])
    mask = (far > near).to(torch.float32).sum(-1)
    return torch.where(mask > 0)[0].to(torch.int32).cpu().tolist()


def build_tree_nodes(c2w, intri, bounds, bbox_levels, max_level, split_dist_thres):
    """ConstructTreeNode (PersSampler.cpp:359-421) without ConstructTrans: the initial octree of the training cameras as
    ``TreeNode`` records, a numpy array of ``TREE_NODE`` (zero padding; the reference leaves its padding uninitialised).

    ``c2w`` [n,3,4], ``intri`` [n,3,3], ``bounds`` [n,2]: the training cameras (``Dataset::c2w_train_`` etc.), float32 on
    the device the visibility tests should run on.  The root is the cube of side ``2^(bbox_levels-1)`` at the origin; a node
    splits while at least N_PROS / 2 cameras see it and the DistanceSummary of their distances is below
    ``side_len * split_dist_thres``, down to depth ``max_level``.  Nodes are numbered as the reference allocates them:
    the recursion enters each child right after appending it.  A leaf seen by N_PROS / 2 cameras or more is valid and
    gets the next ``trans_idx``."""
    c2w = c2w.to(torch.float32).contiguous()
    bounds = bounds.to(torch.float32).contiguous()
    intri0 = intri[0].to(torch.float32)
    dev = c2w.device
    cam_pos = c2w[:, 0:3, 3].contiguous()
    split = f32(split_dist_thres)
    nodes = []
    n_trans = [0]

    def new_node():
        nodes.append(np.zeros((), TREE_NODE))
        return len(nodes) - 1

    def construct(u, depth, center, side_len):
        node = nodes[u]
        node["center"], node["side_len"], node["is_leaf"], node["trans_idx"] = center, side_len, 0, -1
        node["childs"] = -1
        if depth > max_level:
            node["is_leaf"] = 1
            return
        center_ts = torch.from_numpy(center.copy()).to(dev)
        visi = visible_cams(side_len, center_ts, c2w, intri0, bounds)
        cam_dis = torch.linalg.norm(cam_pos - center_ts.unsqueeze(0), 2, -1, True).cpu().reshape(-1)
        summary = distance_summary(cam_dis[visi].to(dev))
        if len(visi) >= N_PROS // 2 and summary < f32(side_len) * split:
            half = f32(side_len) * f32(.5)
            for st in range(8):
                v = new_node()
                offset = np.array([((st >> 2) & 1), ((st >> 1) & 1), (st & 1)], np.float32) - f32(.5)
                nodes[u]["childs"][st] = v
                nodes[v]["parent"] = u
                construct(v, depth + 1, center + half * offset, half)
        elif len(visi) < N_PROS // 2:
            node["is_leaf"] = 1                     # a leaf without enough cameras to hold a warp
        else:
            node["is_leaf"] = 1
            node["trans_idx"] = n_trans[0]
            n_trans[0] += 1

    # The reference's ray directions come from a full-float32 matmul (LibTorch's default).  A process that enabled TF32 would
    # round them differently and could flip visibility decisions, so TF32 is off for the build and restored afterwards.  The
    # flag is process-wide: do not run other CUDA matmuls on other threads meanwhile.
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        root = new_node()
        nodes[root]["parent"] = -1
        construct(root, 0, np.zeros(3, np.float32), f32(1 << (int(bbox_levels) - 1)))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32
    out = np.zeros(len(nodes), TREE_NODE)
    for name in TREE_NODE.names:
        out[name] = [n[name] for n in nodes]
    return out


def build_edge_pool(tree_nodes, chunk_pairs=1 << 20):
    """ConstructEdgePool (PersSampler.cpp:614-659): for every pair of valid leaves (a, b), a < b in node order, the faces
    of the smaller one whose centre lies inside the other (``max |(pt - c) / s * 2| < 1 + 1e-4``), in the reference's push
    order (+x, -x, +y, -y, +z, -z).  ``tree_nodes``: TREE_NODE records or their bytes.  Returns EDGE_POOL records (zero
    padding, as the reference's)."""
    nodes = np.ascontiguousarray(tree_nodes).view(np.uint8).reshape(-1).view(TREE_NODE)
    valid = np.nonzero(nodes["trans_idx"] >= 0)[0]
    n = len(valid)
    rows = max(1, int(chunk_pairs) // max(n, 1))    # pairs go in chunks of `a` (push order kept): bounded memory
    chunks = [_edge_pool_pairs(nodes, valid, start, min(start + rows, n)) for start in range(0, n, rows)]
    out = np.zeros(sum(len(c) for c in chunks), EDGE_POOL)    # (np.concatenate would pack the records to 44 bytes)
    pos = 0
    for c in chunks:
        out[pos:pos + len(c)] = c
        pos += len(c)
    return out


def _edge_pool_pairs(nodes, valid, start, stop):
    """The edge records of the pairs (valid[i], valid[j]) with start <= i < stop and j > i, in push order."""
    ia, ib = np.nonzero(np.arange(len(valid))[None, :] > np.arange(start, stop)[:, None])    # row-major: a, then b ascending
    a, b = valid[ia + start], valid[ib]
    side, center = nodes["side_len"], nodes["center"]
    swap = side[a] > side[b]
    u, v = np.where(swap, b, a), np.where(swap, a, b)
    len_u = side[u] * f32(.5)                                                   # [P]
    ct_u, ct_v, s_v = center[u][:, None, :], center[v][:, None, :], side[v][:, None, None]
    axis = np.repeat(np.eye(3, dtype=np.float32), 2, axis=0)                     # face k: axis k // 2
    step = len_u[:, None, None] * axis[None]                                    # [P, 6, 3]: len_u on the axis, +0 elsewhere
    plus = (np.arange(6) % 2 == 0)[None, :, None]
    pts = np.where(plus, ct_u + step, ct_u - step)
    bias = (pts - ct_v) / s_v * f32(2.)
    inside = np.abs(bias).max(-1) < f32(1.) + f32(1e-4)                          # [P, 6]
    dir_axes = np.array([[1, 2], [1, 2], [0, 2], [0, 2], [0, 1], [0, 1]])       # the face's two tangent axes
    out = np.zeros(int(inside.sum()), EDGE_POOL)
    p, k = np.nonzero(inside)                                                    # pair-major, face-minor: the push order
    out["t_idx_a"], out["t_idx_b"] = nodes["trans_idx"][a[p]], nodes["trans_idx"][b[p]]
    out["center"] = pts[p, k]
    eye = np.eye(3, dtype=np.float32)
    out["dir_0"] = len_u[p, None] * eye[dir_axes[k, 0]]
    out["dir_1"] = len_u[p, None] * eye[dir_axes[k, 1]]
    return out


def initial_octree(dataset, pts_sampler_cfg):
    """(tree_nodes, edge_pool) records of the initial octree of ``dataset``'s training cameras under a ``pts_sampler``
    config (``bbox_levels``, ``max_level``, ``split_dist_thres``), as PersSampler's constructor builds them
    (PersSampler.cpp:664-690), on the dataset's device."""
    idx = torch.tensor(dataset.train_set_, dtype=torch.long, device=dataset.poses_.device)
    c2w, intri, bounds = (t.index_select(0, idx).contiguous() for t in (dataset.poses_, dataset.intri_, dataset.bounds_))
    nodes = build_tree_nodes(c2w, intri, bounds, int(pts_sampler_cfg["bbox_levels"]), int(pts_sampler_cfg["max_level"]),
                             float(f32(pts_sampler_cfg["split_dist_thres"])))
    return nodes, build_edge_pool(nodes)
