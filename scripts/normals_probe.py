"""Timing of the surface-normal queries (DESIGN.md §3j) on the ngp_fox scene (the reference's octree and warps from
tests/golden, the test suite's deterministic field parameters):
- geometry.QueryGradient against geometry.QueryLogit at 2^20 and 2^24 world points spread over the valid leaves;
- eval.RenderNormals against eval.RenderWholeImage per 960 x 540 view (the 7 test cameras of tests/golden/ref_ngp_fox_camrays.npz).
CUDA events; medians over --reps after one warm-up.  The card's name and power limit are read in the same run.

    python scripts/normals_probe.py [--reps 5] [--out profiles/h100_normals_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                                            # noqa: BLE001  (no nvidia-smi: say so in the record)
        return None


def main():
    import numpy as np
    import torch
    from f2nerf_b200 import RayGenerator, RenderNormals, RenderWholeImage
    from f2nerf_b200 import geometry as G
    from f2nerf_b200.octree_build import TREE_NODE
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_normals_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, sb = make_renderer()
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = ev(), ev()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    nd = sb["nodes"].view(TREE_NODE)
    leaf = np.nonzero((nd["trans_idx"] >= 0) & (nd["childs"] < 0).all(1))[0]
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, points={}, views={})
    for lg in (20, 24):
        n = 1 << lg
        g = torch.Generator(device="cuda").manual_seed(lg)
        pick = torch.as_tensor(leaf, device="cuda")[torch.randint(0, len(leaf), (n,), generator=g, device="cuda")]
        c = torch.as_tensor(nd["center"], device="cuda")[pick]
        s = torch.as_tensor(nd["side_len"], device="cuda")[pick, None]
        pts = (c + (torch.rand((n, 3), generator=g, device="cuda") - .5) * .98 * s).contiguous()
        t_logit = timed(lambda: G.QueryLogit(renderer, pts))
        t_grad = timed(lambda: G.QueryGradient(renderer, pts))
        out["points"][f"2^{lg}"] = dict(query_logit_ms=t_logit, query_gradient_ms=t_grad, ratio=t_grad / t_logit,
                                         gradient_points_per_s=n / (t_grad * 1e-3))
        del pts
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    cams = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    gen = RayGenerator(d["ds_poses"].reshape(-1, 3, 4)[cams], d["ds_intri"].reshape(-1, 3, 3)[cams], d["ds_dist_params"][cams],
                       d["ds_bounds"][cams], height=H, width=W, test_set=range(len(cams)))
    per = []
    for i in range(len(cams)):
        o, dd, _ = gen.RaysOfCamera(i)
        o, dd = o.cuda().contiguous(), dd.cuda().contiguous()
        t_img = timed(lambda: RenderWholeImage(renderer, o, dd))
        t_nrm = timed(lambda: RenderNormals(renderer, o, dd))
        per.append((t_img, t_nrm))
    a = np.asarray(per)
    out["views"] = dict(height=H, width=W, n_views=len(cams), render_whole_image_ms=float(np.median(a[:, 0])),
                        render_normals_ms=float(np.median(a[:, 1])), ratio=float(np.median(a[:, 1] / a[:, 0])))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
