"""CPU checks of the initial-octree rebuild that lets a reference checkpoint resume training (f2nerf_b200/octree_build.py,
checkpoint.load_scene(trainable=True)):
- the edge-pool port on the reference's initial ngp_fox tree (tests/golden/ref_ngp_fox.npz) reproduces its edge pool byte
  for byte;
- the structure builder, fed the same fixture's training cameras on CPU torch, reproduces the reference's initial tree in
  every field (the padding, which the reference never initialises, excepted).  The reference ran these ops on CUDA; CPU
  ATen may round the scalar divisions and the batched matmul differently, but on this scene no visibility decision flips.
  tests/test_gpu_checkpoint_resume.py pins the device result from the data directory;
- ``gradient_scaling_progress`` as ``ExpRunner::UpdateAdaParams`` computes it;
- the ValueErrors of a rebuilt tree that does not fit the checkpoint's warps."""
import numpy as np
import pytest
import torch
import yaml

from f2nerf_b200 import build_edge_pool, build_tree_nodes, gradient_scaling_progress, load_scene
from f2nerf_b200.checkpoint import check_initial_octree
from f2nerf_b200.octree_build import EDGE_POOL, TREE_NODE
from test_checkpoint_cpu import GOLDEN, FOX_CONFIG, make_experiment

FOX_GOLDEN = f"{GOLDEN}/ref_ngp_fox.npz"
FOX_SAMPLER = dict(bbox_levels=10, max_level=16, split_dist_thres=1.5)        # oracle/ref_config_ngp_fox.yaml


def golden():
    return np.load(FOX_GOLDEN)


def fields_mask():
    """The bytes of a TreeNode that hold a field: all but 53..55 and 60..63."""
    m = np.zeros(64, bool)
    for name in TREE_NODE.names:
        dt, off = TREE_NODE.fields[name]
        m[off:off + dt.itemsize] = True
    return m


def golden_cameras():
    z = golden()
    c2w = torch.from_numpy(z["ds_poses"][z["ds_train_set"]].reshape(-1, 3, 4).copy())
    return c2w, torch.from_numpy(z["oct_intri"].reshape(-1, 3, 3).copy()), torch.from_numpy(z["oct_bound"].copy())


@pytest.fixture(scope="module")
def fox_tree_cpu():
    c2w, intri, bounds = golden_cameras()
    return build_tree_nodes(c2w, intri, bounds, **FOX_SAMPLER)


def test_record_layouts():
    assert TREE_NODE.itemsize == 64 and EDGE_POOL.itemsize == 64
    assert fields_mask().sum() == 12 + 4 + 4 + 32 + 1 + 4


def test_edge_pool_matches_reference():
    z = golden()
    pool = build_edge_pool(z["tree_nodes"])
    assert len(pool) == 1131
    assert np.array_equal(pool.view(np.uint8).reshape(-1), z["edge_pool"])
    chunked = build_edge_pool(z["tree_nodes"], chunk_pairs=1000)     # 2 rows of `a` per chunk: same records, same order
    assert np.array_equal(chunked.view(np.uint8).reshape(-1), z["edge_pool"])


def test_edge_pool_of_two_face_neighbours():
    """Two valid leaves of side 2 and 1 sharing the x = 1 plane: one record, the smaller leaf's -x face, indices in node
    order (not the swapped order of the size test)."""
    nodes = np.zeros(2, TREE_NODE)
    nodes["center"] = [[0, 0, 0], [1.5, .5, -.5]]
    nodes["side_len"] = [2, 1]
    nodes["trans_idx"] = [7, 3]
    pool = build_edge_pool(nodes)
    assert len(pool) == 1
    r = pool[0]
    assert (r["t_idx_a"], r["t_idx_b"]) == (7, 3)
    assert r["center"].tolist() == [1., .5, -.5] and r["dir_0"].tolist() == [0, .5, 0] and r["dir_1"].tolist() == [0, 0, .5]
    nodes["trans_idx"][1] = -1                                       # an invalid leaf takes no part
    assert len(build_edge_pool(nodes)) == 0


def test_tree_structure_matches_reference_on_cpu(fox_tree_cpu):
    want = golden()["tree_nodes"].reshape(-1, 64)
    got = fox_tree_cpu.view(np.uint8).reshape(-1, 64)
    assert got.shape == want.shape == (897, 64)
    m = fields_mask()
    assert np.array_equal(got[:, m], want[:, m])
    assert not got[:, ~m].any()                                      # zero padding
    assert (fox_tree_cpu["trans_idx"] >= 0).sum() == 372


def test_rebuilt_tree_fits_reference_warps(fox_tree_cpu):
    z = golden()
    check_initial_octree(fox_tree_cpu, z["pers_trans"], fox_cfg())
    assert np.array_equal(build_edge_pool(fox_tree_cpu).view(np.uint8).reshape(-1), z["edge_pool"])


def fox_cfg(**pts_sampler):
    with open(FOX_CONFIG) as f:
        cfg = yaml.safe_load(f)
    cfg["pts_sampler"].update(pts_sampler)
    return cfg


def test_wrong_split_dist_thres_is_refused():
    """A tree from another split_dist_thres has other leaves than the checkpoint's warps.  (0.5 splits far less than 1.5,
    which keeps this build short.)"""
    c2w, intri, bounds = golden_cameras()
    nodes = build_tree_nodes(c2w, intri, bounds, **dict(FOX_SAMPLER, split_dist_thres=.5))
    with pytest.raises(ValueError, match="split_dist_thres = 0.5"):
        check_initial_octree(nodes, golden()["pers_trans"], fox_cfg(split_dist_thres=.5))


def test_warp_centre_mismatch_is_refused(fox_tree_cpu):
    trans = golden()["pers_trans"].copy().reshape(-1, 544)
    centre = trans[5, 528:540].view(np.float32)
    centre[1] = np.nextafter(centre[1], np.float32(np.inf))          # one ulp: the check is bit for bit
    with pytest.raises(ValueError, match="warp 5 is centred at"):
        check_initial_octree(fox_tree_cpu, trans.reshape(-1), fox_cfg())


def test_warp_count_mismatch_is_refused(fox_tree_cpu):
    trans = golden()["pers_trans"].reshape(-1, 544)[:-1]
    with pytest.raises(ValueError, match="371 warps.*ngp_fox has 372 valid leaves"):
        check_initial_octree(fox_tree_cpu, trans, fox_cfg())


def test_load_scene_trainable_refuses_checkpoint_of_another_scene(tmp_path):
    """The fixture archive's two warps on a five-camera directory: fewer than N_PROS / 2 cameras see the root, so the
    initial octree has no valid leaf."""
    conf = make_experiment(tmp_path)
    with pytest.raises(ValueError, match=r"2 warps.*dataset.data_path = .*data has 0 valid leaves"):
        load_scene(conf, device="cpu", trainable=True)
    assert load_scene(conf, device="cpu").renderer.pts_sampler_.n_edges == 0       # the default still loads it


def test_gradient_scaling_progress_values():
    """The ramp of the ngp_fox config (gradient_scaling_start 1000, end 5000).  1e-9f vanishes next to 4000 in float, so
    each value is the float nearest (iter - 1000) / 4000.  tests/test_gpu_checkpoint_resume.py pins the resumed value
    against the reference program."""
    assert gradient_scaling_progress(300, 1000, 5000) == 0.0                        # before the start: clamped at 0
    assert gradient_scaling_progress(5000, 1000, 5000) == 1.0 == gradient_scaling_progress(9000, 1000, 5000)
    for it, want in ((1000, 0.0), (2000, 0.25), (3000, 0.5), (4000, 0.75), (1001, 0.0002500000118743628),
                     (4999, 0.9997500181198120)):
        assert gradient_scaling_progress(it, 1000, 5000) == want, it
    assert gradient_scaling_progress(10, 0, 3) == 1.0 and gradient_scaling_progress(1, 0, 3) == 0.3333333432674408
