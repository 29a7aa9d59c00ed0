"""CPU checks of the reference-checkpoint and data-directory loaders (f2nerf_b200/checkpoint.py, dataset.load_dataset):
- the archive reader against tests/golden/libtorch_states.pt / libtorch_scalars.pt, written by LibTorch's own torch::save
  (oracle/make_golden_checkpoint.cpp, whose values are restated in ``fixture_states``);
- ``load_dataset`` on the reference's ngp_fox example (oracle/_ref/data, made by oracle/Makefile.ref's data target; skipped
  without it) against the reference program's own tensors in tests/golden: within 2 ulp, since CPU and CUDA reductions may
  order their sums differently (tests/test_gpu_checkpoint.py pins the device result bit for bit);
- ``load_scene`` on a small synthetic data directory with the fixture archive as its checkpoint, and its error paths."""
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

from f2nerf_b200 import VALIDATE, load_dataset, load_scene, load_states
from f2nerf_b200.checkpoint import load_iter_step, ray_march_fineness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FOX = os.path.join(ROOT, "oracle", "_ref", "data", "ngp_fox")
FOX_CONFIG = os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml")
need_fox = pytest.mark.skipif(not os.path.isfile(os.path.join(FOX, "image_list.txt")),
                              reason="oracle/_ref/data/ngp_fox not built (make -f oracle/Makefile.ref data)")
FIXTURE_V, FIXTURE_LOG2, FIXTURE_IMAGES = 2, 4, 5


def fixture_states():
    """What oracle/make_golden_checkpoint.cpp saves, restated in numpy."""
    u8 = lambda n, mul, add: ((np.arange(n) * mul + add) % 256).astype(np.uint8)
    f32 = lambda shape, mul: (((np.arange(int(np.prod(shape))) * mul) % 2001 - 1000).astype(np.float32) / np.float32(1024)).reshape(shape)
    V = FIXTURE_V
    return [u8(2 * 64, 37, 11), u8(V * 544, 13, 5), np.array([3, -7], np.int32),
            np.array([2000, 4000, 6000, 8000, 10000], np.int32), f32(((1 << FIXTURE_LOG2) * 16, 2), 7919),
            ((1 << 28) + 7 * np.arange(16 * V * 3)).astype(np.int32).reshape(16, V, 3), f32((16 * V, 3), 104729),
            np.array([V], np.int32), f32((32 * 64 + 64 * 16,), 31), f32((32 * 64 + 64 * 64 + 64 * 16,), 17),
            f32((FIXTURE_IMAGES, 16), 523)]


def assert_same_states(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        g = g.detach().cpu().numpy() if isinstance(g, torch.Tensor) else g
        w = w.detach().cpu().numpy() if isinstance(w, torch.Tensor) else w
        assert g.dtype == w.dtype and g.shape == w.shape, (i, g.dtype, g.shape, w.dtype, w.shape)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), i


def test_load_states_reads_libtorch_archive():
    states = load_states(os.path.join(GOLDEN, "libtorch_states.pt"), "cpu")
    assert len(states) == 11                                     # keys "0".."10": "10" sorts before "2" as a string
    assert_same_states(states, fixture_states())
    assert all(not t.requires_grad for t in states)


def test_load_iter_step_reads_scalars():
    assert load_iter_step(os.path.join(GOLDEN, "libtorch_scalars.pt")) == 1234


def test_load_states_missing_file(tmp_path):
    with pytest.raises(FileNotFoundError):
        load_states(str(tmp_path / "renderer.pt"), "cpu")


def test_ray_march_fineness_is_float_arithmetic():
    assert ray_march_fineness(10000, 16., 10000) == 1.0 and ray_march_fineness(20000, 16., 10000) == 1.0
    for it in (0, 1, 300, 5000, 9999):
        v = ray_march_fineness(it, 16., 10000)
        assert float(np.float32(v)) == v                         # a float result, as the reference stores it
        p = it / 10000
        assert abs(v - np.exp(np.log(16.) * (1 - p))) <= 4 * np.spacing(np.float32(v))


# ---- load_dataset on the reference's ngp_fox example ------------------------------------------------------------------

def assert_ulp(got, want, maxulp=2):
    got = np.ascontiguousarray(got, np.float32)
    np.testing.assert_array_max_ulp(got, np.ascontiguousarray(want, np.float32).reshape(got.shape), maxulp=maxulp)


@pytest.fixture(scope="module")
def fox_cpu():
    return load_dataset(FOX, 2, [0.5, 4.0], "cpu")


@need_fox
def test_load_dataset_matches_reference_tables(fox_cpu):
    ds = fox_cpu
    run = np.load(os.path.join(GOLDEN, "ref_ngp_fox_run.npz"))
    cam = np.load(os.path.join(GOLDEN, "ref_ngp_fox_camrays.npz"))
    assert_ulp(ds.poses_.reshape(-1, 12).numpy(), run["ds_poses"])
    assert_ulp(ds.intri_.reshape(-1, 9).numpy(), run["ds_intri"])
    assert_ulp(ds.dist_params_.numpy(), run["ds_dist_params"])
    assert_ulp(ds.bounds_.numpy(), run["ds_bounds"])
    assert_ulp(ds.render_poses_.reshape(-1, 12).numpy(), cam["cam_render_poses"])
    assert (ds.height_, ds.width_) == tuple(int(v) for v in run["ds_hw"])
    assert ds.train_set_ == run["ds_train_set"].tolist()
    assert ds.test_set_ == cam["cam_test_set"].tolist() and ds.val_set_ == []


@need_fox
def test_load_dataset_ground_truth_pixels(fox_cpu):
    """PIL (libjpeg) against the reference's stb_image at the 512 pixels of the reference's ray batch: at most 2 levels."""
    rays = np.load(os.path.join(GOLDEN, "ref_ngp_fox_512_rays.npz"))
    cam, ij = rays["emb_idx"].astype(np.int64), rays["ray_ij"].astype(np.int64)
    got = fox_cpu.image_tensors_[cam, ij[:, 0], ij[:, 1]].numpy()
    assert np.abs(got - rays["gt_colors"]).max() <= 2 / 255 + 1e-6
    levels = got * np.float32(255)
    assert np.abs(levels - np.rint(levels)).max() < 1e-4      # u8 / 255: every value is a whole level


# ---- load_scene on a synthetic data directory with the fixture archive --------------------------------------------------

def make_data_dir(path, n_images, hw=(12, 16), split=None, image_list=False):
    """A reference data directory of ``n_images`` cameras around the origin with PNG images under images_2/."""
    from PIL import Image
    rng = np.random.default_rng(n_images)
    os.makedirs(os.path.join(path, "images_2"), exist_ok=True)
    meta = np.zeros((n_images, 27), np.float64)
    for i in range(n_images):
        a = 2 * np.pi * i / n_images
        c2w = np.array([[np.cos(a), 0, np.sin(a), 3 * np.sin(a)], [0, 1, 0, .2 * i], [-np.sin(a), 0, np.cos(a), 3 * np.cos(a)]])
        meta[i, :12] = c2w.reshape(-1)
        meta[i, 12:21] = [20., 0, hw[1], 0, 20., hw[0], 0, 0, 1]
        meta[i, 25:27] = [.5 + .01 * i, 9.]
    np.save(os.path.join(path, "cams_meta.npy"), meta)
    names = []
    for i in range(n_images):
        name = os.path.join(path, "images_2", f"{i:04d}.png")
        Image.fromarray(rng.integers(0, 256, (*hw, 3), dtype=np.uint8)).save(name)
        names.append(name)
    if split is not None:
        np.save(os.path.join(path, "split.npy"), np.asarray(split, np.uint8))
    if image_list:                                               # data-directory-relative entries, reversed order
        with open(os.path.join(path, "image_list.txt"), "w") as f:
            f.writelines(os.path.relpath(n, path) + "\n" for n in reversed(names))
    return names


def make_experiment(tmp_path, n_images=FIXTURE_IMAGES, log2=FIXTURE_LOG2):
    """config + data directory + checkpoints/latest holding the fixture archive -> config path."""
    data = str(tmp_path / "data")
    make_data_dir(data, n_images)
    with open(FOX_CONFIG) as f:
        cfg = yaml.safe_load(f)
    cfg["base_exp_dir"] = str(tmp_path / "exp")
    cfg["dataset"]["data_path"] = data
    cfg["field"]["log2_table_size"] = log2
    ck = tmp_path / "exp" / "checkpoints" / "latest"
    ck.mkdir(parents=True)
    shutil.copy(os.path.join(GOLDEN, "libtorch_states.pt"), ck / "renderer.pt")
    shutil.copy(os.path.join(GOLDEN, "libtorch_scalars.pt"), ck / "scalars.pt")
    conf = tmp_path / "runtime_config.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    return str(conf)


def test_load_dataset_split_and_image_list(tmp_path):
    names = make_data_dir(str(tmp_path), 6, split=[1, 2, 1, 4 | 1, 2, 3], image_list=True)
    ds = load_dataset(str(tmp_path), 2., [.5, 4.], "cpu")
    assert (ds.train_set_, ds.test_set_, ds.val_set_) == ([0, 2, 3, 5], [1, 4, 5], [3])
    from PIL import Image
    first = np.asarray(Image.open(names[-1])).astype(np.float32) / np.float32(255)      # image_list.txt is reversed
    assert np.array_equal(ds.image_tensors_[0].numpy(), first)
    assert (ds.height_, ds.width_) == (12, 16)
    assert float(ds.bounds_.min()) >= 1e-2


def test_load_dataset_default_split(tmp_path):
    make_data_dir(str(tmp_path), 10)
    ds = load_dataset(str(tmp_path), 2., [.5, 4.], "cpu")
    assert ds.test_set_ == [0, 8] and ds.train_set_ == [1, 2, 3, 4, 5, 6, 7, 9]
    assert ds.render_poses_ is None
    assert torch.allclose(ds.poses_[:, :, 3].mean(0), torch.zeros(3), atol=1e-6)
    assert abs(float(torch.linalg.norm(ds.poses_[:, :, 3], 2, -1).max()) - 1.) < 1e-6


def test_load_scene_on_cpu(tmp_path):
    scene = load_scene(make_experiment(tmp_path), device="cpu")
    gdp, renderer, ds, iter_step = scene
    assert iter_step == 1234 and gdp.iter_step_ == 1234 and gdp.mode_ == VALIDATE
    assert gdp.ray_march_fineness_ == ray_march_fineness(1234, 16., 10000) and gdp.ray_march_fineness_ > 1.
    assert ds.n_images_ == FIXTURE_IMAGES and gdp.n_volumes_ == FIXTURE_V
    assert renderer.scene_field_.local_size_ == 1 << FIXTURE_LOG2
    assert_same_states(renderer.States(), fixture_states())
    assert renderer.pts_sampler_.global_near_ == float(np.float32(.01))
    assert renderer.pts_sampler_.n_edges == 0                  # no edge pool in a reference checkpoint: evaluation only


def test_load_scene_wrong_table_size(tmp_path):
    with pytest.raises(ValueError, match="log2_table_size"):
        load_scene(make_experiment(tmp_path, log2=19), device="cpu")


def test_load_scene_wrong_image_count(tmp_path):
    with pytest.raises(ValueError, match="image count"):
        load_scene(make_experiment(tmp_path, n_images=FIXTURE_IMAGES + 1), device="cpu")


def test_load_scene_missing_files(tmp_path):
    conf = make_experiment(tmp_path)
    with pytest.raises(FileNotFoundError):
        load_scene(conf, checkpoint_dir=str(tmp_path / "nowhere"), device="cpu")
    with pytest.raises(FileNotFoundError):
        load_scene(str(tmp_path / "missing.yaml"), device="cpu")
    os.remove(tmp_path / "data" / "images_2" / "0003.png")
    with pytest.raises(ValueError, match="4 images"):
        load_scene(conf, device="cpu")
