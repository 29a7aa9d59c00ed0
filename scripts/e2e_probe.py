"""Where the end-to-end step (host rays in, loss out) spends its wall time: host-side stopwatch around every phase of
bench.train_step inside the e2e loop of bench.py (upload -> Render -> prefetch -> loss -> backward -> loss.item()).

    python scripts/e2e_probe.py [--config wanjinyou] [--steps 12] [--no-pipeline-march] > gpurun_out/e2e_probe.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import bench
    from f2nerf_b200 import CustomOps
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="wanjinyou")
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--rays", type=int, default=0)
    ap.add_argument("--no-pipeline-march", dest="pipeline_march", action="store_false")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    prob = bench.build_problem(0, 1, args, dev)
    o, d, cam, gt = prob["host"]
    pin = lambda a: torch.from_numpy(a).pin_memory()
    h_o, h_d, h_cam, h_gt = pin(o), pin(d), pin(cam), pin(gt)
    r = prob["renderer"]
    up = lambda: (h_o.to(dev, non_blocking=True), h_d.to(dev, non_blocking=True))
    rows = []
    ro, rd = up()
    torch.cuda.synchronize()
    for it in range(args.steps + 4):
        seg = {}
        t = time.perf_counter()

        def lap(name):
            nonlocal t
            n = time.perf_counter()
            seg[name] = round((n - t) * 1e3, 3)
            t = n

        t_step = t
        rc, rg = h_cam.to(dev, non_blocking=True), h_gt.to(dev, non_blocking=True)
        for p in (prob["field"].feat_pool_, prob["field"].mlp_.params_, prob["shader"].mlp_.params_, r.app_emb_):
            p.grad = None
        lap("upload_cam_gt")
        res = r.Render(ro, rd, None, rc)
        lap("render")
        if args.pipeline_march:
            nxt = up()
            r.prefetch_next(nxt[0], nxt[1])
        lap("prefetch")
        color_loss = torch.sqrt((res.colors - rg) ** 2 + 1e-4).mean()
        var_loss = torch.sqrt(CustomOps.WeightVar(res.weights, res.idx_start_end) + 1e-2).mean()
        tv_loss = ((res.edge_feats[:, 0] - res.edge_feats[:, 1]) ** 2).mean()
        loss = color_loss + var_loss * 1e-2 + tv_loss * 1e-1
        lap("loss")
        loss.backward()
        lap("backward_enqueue")
        v = float(loss.item())
        lap("loss_item_sync")
        if args.pipeline_march:
            ro, rd = nxt
        else:
            ro, rd = up()
        seg["step"] = round((time.perf_counter() - t_step) * 1e3, 3)
        if it >= 4:
            rows.append(seg)
    keys = rows[0].keys()
    med = {k: sorted(x[k] for x in rows)[len(rows) // 2] for k in keys}
    print(json.dumps({"config": args.config, "pipeline_march": args.pipeline_march, "median_ms": med, "rows": rows[:6],
                      "n_kept": r.n_kept_pts_}))


if __name__ == "__main__":
    main()
