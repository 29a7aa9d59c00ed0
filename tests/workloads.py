"""Workload definitions shared by bench.py, the headline-size parity tests and smoke().  numpy/torch-CPU only:
importing this module does NOT load libf2nerf_b200.so, so bench.py's `--impl reference` (CPU) arm can use it.

BASELINE.json `configs` -> the reference YAMLs they name (sampler / renderer / field settings that reach the path):

  wanjinyou  configs[1]  confs/wanjinyou.yaml:21-27      near 0.01, scale_by_dis, use_app_emb, log2_table_size 19, 4096 rays (headline)
  free       configs[2]  confs/free.yaml + defaults       near 0.05, scale_by_dis false, no app-emb (confs/pts_sampler/perspective.yaml:11-12,
                                                          confs/renderer/default.yaml:2), log2 19
  nerf360    configs[3]  confs/nerf-360.yaml + defaults   same sampler as free; 8192 rays GLOBAL, split over the ranks (strong scaling)
  big20      configs[4]  confs/wanjinyou_big.yaml:18-19   wanjinyou + log2_table_size 20 (what the YAML says)
  big22      configs[4]  BASELINE.json's "2^22 entries"   wanjinyou + log2_table_size 22 (table no longer L2-resident)
  synthetic  (round 1)   wanjinyou sampler on the synthetic 24-camera octree of tests/synth_scene.py

Scene: the only dataset the reference ships is data/example/ngp_fox; its octree / warp / edge blobs, cameras and hash
primes / biases as the UNMODIFIED reference built them are committed in tests/golden/ref_ngp_fox.npz (oracle/make_golden.py; kept
fixed so the benchmark's inputs do not move), while the reference-parity tests use a later run of the reference: the scene it built
(tests/golden/ref_ngp_fox_run.npz: the same octree, warp weights equal to ~1e-7, its own random biases) and the dumps of a small
seeded ray batch through it (tests/golden/ref_ngp_fox_rays.npz) and of its optimizer step (tests/golden/ref_ngp_fox_adam.npz),
so every config runs on the reference's own ngp_fox geometry with that config's settings.  Rays are drawn like
Dataset::RandRaysData (Dataset.cpp:287-289: camera / row / column from the CPU generator) so the compiled reference
(oracle/_ref/ref_driver, seed 2023) marches the very same batch.  Parameters are initialised like oracle/ref_driver.cpp:76-83
(table U(-1,1) from CPU generator 1234, field MLP x4, appearance embedding from the same generator).
"""
import os
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox.npz")
GOLD_RUN = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_run.npz")
GOLD_RAYS = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_rays.npz")
GOLD_ADAM = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_adam.npz")

_W = dict(near=0.01, scale_by_dis=True, use_app_emb=True, sample_l=1.0 / 256)
_F = dict(near=0.05, scale_by_dis=False, use_app_emb=False, sample_l=1.0 / 256)
CONFIGS = {
    "wanjinyou": dict(_W, log2_table=19, rays=4096, scaling="weak", scene="ngp_fox", ref_yaml="oracle/ref_config_ngp_fox.yaml",
                      baseline_config=1, yaml="confs/wanjinyou.yaml"),
    "free": dict(_F, log2_table=19, rays=4096, scaling="weak", scene="ngp_fox", ref_yaml="oracle/ref_config_free.yaml",
                 baseline_config=2, yaml="confs/free.yaml"),
    "nerf360": dict(_F, log2_table=19, rays=8192, scaling="strong", scene="ngp_fox", ref_yaml="oracle/ref_config_free.yaml",
                    baseline_config=3, yaml="confs/nerf-360.yaml"),
    "big20": dict(_W, log2_table=20, rays=4096, scaling="weak", scene="ngp_fox", ref_yaml="oracle/ref_config_big20.yaml",
                  baseline_config=4, yaml="confs/wanjinyou_big.yaml"),
    "big22": dict(_W, log2_table=22, rays=4096, scaling="weak", scene="ngp_fox", ref_yaml="oracle/ref_config_big22.yaml",
                  baseline_config=4, yaml="confs/wanjinyou_big.yaml + BASELINE.json's 2^22"),
    "synthetic": dict(_W, log2_table=19, rays=4096, scaling="weak", scene="synthetic", ref_yaml=None, baseline_config=1,
                      yaml="confs/wanjinyou.yaml"),
}


def load_ngp_fox():
    """The reference's ngp_fox scene as committed: dict with tree_nodes / pers_trans / edge_pool (u8 blobs), prim_pool,
    bias_pool, ds_poses [n,12], ds_intri [n,9], ds_dist_params, ds_bounds, ds_hw, ds_train_set, scalars, level_scales."""
    g = dict(np.load(GOLD))
    return g


def diag_path(name):
    """Where a test writes its diagnostics (JSON summaries, subprocess logs): a directory under the system's temporary
    directory, so that the suite also runs on a read-only tree."""
    d = os.path.join(tempfile.gettempdir(), "f2b_test_diag")
    os.makedirs(d, exist_ok=True)
    return os.path.join(d, name)


def load_golden(batch="ref_ngp_fox"):
    """A reference-parity fixture (oracle/make_golden.py): the scene of the reference run, its dumps of the seeded ray batch and
    a sample of its optimizer step, in one dict.  ``batch``: "ref_ngp_fox" (8 rays, every per-sample tensor) or
    "ref_ngp_fox_512" (512 rays, per-sample tensors of the rays listed in ``sample_rays``) or "ref_free_512" (that batch under the
    free config's settings, without an optimizer sample)."""
    d = os.path.join(ROOT, "tests", "golden")
    adam = os.path.join(d, batch + "_adam.npz")
    return dict(np.load(os.path.join(d, batch + "_run.npz")), **np.load(os.path.join(d, batch + "_rays.npz")),
                **(np.load(adam) if os.path.exists(adam) else {}))


def scene_blobs(cfg_name):
    """-> dict(nodes, trans, edges, n_images, cams) for the config's scene."""
    cfg = CONFIGS[cfg_name]
    if cfg["scene"] == "synthetic":
        from synth_scene import SyntheticScene
        sc = SyntheticScene(n_cams=24, seed=0)
        nodes, trans, edges = sc.blobs()
        return dict(nodes=nodes, trans=trans, edges=edges, n_images=len(sc.c2w), synthetic=sc, prim=None, bias=None)
    g = load_ngp_fox()
    u8 = lambda a: np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return dict(nodes=u8(g["tree_nodes"]), trans=u8(g["pers_trans"]), edges=u8(g["edge_pool"]), n_images=int(g["scalars"][6]),
                synthetic=None, prim=g["prim_pool"], bias=g["bias_pool"], golden=g)


def draw_pixels(g, n_rays, seed):
    """Dataset::RandRaysData's CPU draws (Dataset.cpp:287-289) -> (cam [n] i32 dataset indices, ij [n,2] i32)."""
    import torch
    train_set = torch.from_numpy(np.asarray(g["ds_train_set"]).astype(np.int64))
    H, W = int(g["ds_hw"][0]), int(g["ds_hw"][1])
    torch.manual_seed(seed)
    cam = train_set[torch.randint(len(train_set), (n_rays,), dtype=torch.int64)]
    i = torch.randint(0, H, (n_rays,), dtype=torch.int64)
    j = torch.randint(0, W, (n_rays,), dtype=torch.int64)
    return cam.to(torch.int32).numpy(), torch.stack([i, j], -1).to(torch.int32).numpy()


def host_rays(cfg_name, n_rays, seed):
    """One ray batch on the HOST (numpy): (rays_o, rays_d un-normalised, cam idx i32).  ngp_fox: the reference's ray
    generation restated by the oracle (bit-exact against the reference, tests/test_golden_ref.py); synthetic: the builder's."""
    sb = scene_blobs(cfg_name)
    if sb["synthetic"] is not None:
        return sb["synthetic"].rays(n_rays, seed=seed)
    import oracle_lib as O
    g = sb["golden"]
    cam, ij = draw_pixels(g, n_rays, seed)
    o, d = O.img2world_rays(g["ds_poses"], g["ds_intri"], g["ds_dist_params"], cam, ij)
    return o, d, cam


def init_params(cfg_name, n_volumes, n_images, prim=None, bias=None):
    """Deterministic, non-trivial parameters as oracle/ref_driver.cpp:76-83 sets them (so the compiled reference and
    every arm here hold identical state): -> dict(table f32 [pool,2], field_mlp f32, shader_mlp f32, app_emb, prim, bias)."""
    import torch
    import oracle_lib as O
    cfg = CONFIGS[cfg_name]
    pool = (1 << cfg["log2_table"]) * 16
    gen = torch.Generator().manual_seed(1234)
    table = (torch.rand((pool, 2), generator=gen) * 2. - 1.).numpy()
    app = (torch.rand((n_images, 16), generator=gen) * .2 - .1).numpy()
    if prim is None:                                          # synthetic scene: any odd 28..30-bit multipliers / U[100,1100) biases
        rng = np.random.default_rng(2022)
        prim = (rng.integers(1 << 28, 1 << 30, size=(16, n_volumes, 3)).astype(np.int32) | 1)
        bias = (rng.random((16 * n_volumes, 3), dtype=np.float32) * 1000 + 100)
    return dict(table=table, field_mlp=O.mlp_init(32, 0) * np.float32(4), shader_mlp=O.mlp_init(32, 1), app_emb=app,
                prim=np.asarray(prim, np.int32), bias=np.asarray(bias, np.float32))
