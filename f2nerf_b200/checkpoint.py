"""Reference checkpoints — the files ``ExpRunner::SaveCheckpoint`` writes (src/ExpRunner.cpp:203-219) and the scene they
describe, loaded for evaluation on the device.

``checkpoints/<iter>/renderer.pt`` is ``torch::save(Renderer::States())``: a TorchScript archive whose parameters are named
"0", "1", ... in state order; ``scalars.pt`` is ``torch::save`` of a one-element float tensor holding the iteration.
``torch.jit.load`` reads both.

``load_scene`` rebuilds what ``ExpRunner``'s constructor + ``LoadCheckpoint`` build (ExpRunner.cpp:17-62,188-201) from the
flat ``runtime_config.yaml`` the reference program reads: the data directory (``dataset.load_dataset``), ``PersSampler``,
``Hash3DAnchored``, ``SHShader`` and ``Renderer`` with the checkpoint's states, and the ray-march fineness of the saved
iteration.  The result renders and evaluates (``eval.TestImages`` / ``RenderPath`` / ``RenderAllImages``).

By default it does not train: the reference's checkpoint holds no edge pool (``PersSampler::States``, PersSampler.cpp:692-701),
so a TRAIN-mode ``Renderer.Render`` on a loaded scene raises (empty edge pool) before it draws the TV-loss points.
``load_scene(..., trainable=True)`` restores what the reference resumes with instead: the edge pool of the initial octree,
rebuilt from the training cameras (``octree_build``), and the saved iteration's gradient-scaling progress.
"""
import ctypes
import ctypes.util
import math
import os
import warnings
from typing import NamedTuple

import numpy as np
import torch

from .dataset import RayGenerator, load_dataset
from .field import N_CHANNELS, N_LEVELS, Hash3DAnchored
from .renderer import Renderer
from .sampler import VALIDATE, GlobalDataPool, PersSampler
from .shader import SHShader

N_RENDERER_STATES = 11          # PersSampler 4 + Hash3DAnchored 5 + SHShader 1 + app_emb 1


def load_states(path, device="cuda"):
    """The tensors of a ``torch::save(std::vector<Tensor>)`` archive, in vector order (by the integer value of the parameter
    name: "10" follows "9"), on ``device``."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"load_states: {path} does not exist")
    with warnings.catch_warnings():                                        # torch.jit.load is deprecated, and the only
        warnings.simplefilter("ignore", DeprecationWarning)                 # reader of LibTorch's torch::save archives
        named = dict(torch.jit.load(path, map_location=torch.device(device)).named_parameters())
    keys = sorted(named, key=int)
    if keys != [str(i) for i in range(len(keys))]:
        raise ValueError(f"load_states: {path} is not a tensor-vector archive (parameter names {keys[:12]})")
    return [named[k].detach() for k in keys]


def load_iter_step(path):
    """``scalars.pt`` -> the saved iteration, ``std::round(scalars[0])`` (ExpRunner.cpp:191)."""
    v = float(load_states(path, "cpu")[0].reshape(-1)[0])
    return int(math.copysign(math.floor(abs(v) + .5), v))                   # std::round: halves away from zero


_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _fn in (_libm.expf, _libm.logf):
    _fn.restype, _fn.argtypes = ctypes.c_float, [ctypes.c_float]


def ray_march_fineness(iter_step, init_fineness, decay_end_iter):
    """``ExpRunner::UpdateAdaParams``' ray-march fineness (ExpRunner.cpp:221-229): expf(logf(1) p + logf(init) (1 - p)) with
    p = float(iter) / float(decay_end), float arithmetic and libm's expf / logf as the reference's float overloads of
    std::exp / std::log call them.  VALIDATE-mode ray noise is ones * fineness, so one ulp here moves every sample."""
    if iter_step >= decay_end_iter:
        return 1.0
    f32 = np.float32
    p = f32(iter_step) / f32(decay_end_iter)
    x = f32(_libm.logf(1.0)) * p + f32(_libm.logf(float(f32(init_fineness)))) * (f32(1.) - p)
    return float(_libm.expf(float(x)))


def gradient_scaling_progress(iter_step, start, end):
    """``ExpRunner::UpdateAdaParams``' gradient-scaling progress (ExpRunner.cpp:245-253): max(0, (float(iter) - start) /
    (end - start + 1e-9f)) in float arithmetic, 1 at or past ``end``.  The TRAIN backward scales the hash-grid gradients
    of near samples by it (GradientScaling), so a resumed run has to start from the saved iteration's value."""
    if iter_step >= end:
        return 1.0
    f32 = np.float32
    start, end = int(start), int(end)
    return float(max(f32(0.), (f32(iter_step) - f32(start)) / (f32(end - start) + f32(1e-9))))


class Scene(NamedTuple):
    global_data_pool: GlobalDataPool
    renderer: Renderer
    dataset: RayGenerator
    iter_step: int


def _mlp_params(d_in, d_hidden, n_hidden_layers):
    """Parameter count of a TCNNWP network (output padded to 16, no biases)."""
    return d_in * d_hidden + d_hidden * d_hidden * (n_hidden_layers - 1) + d_hidden * 16


def check_states(states, cfg, n_images, path="renderer.pt"):
    """Shape and dtype of every ``Renderer::States()`` entry against the config and the data directory; ValueError naming the
    config key that disagrees."""
    if len(states) != N_RENDERER_STATES:
        raise ValueError(f"{path}: {len(states)} states; a PersSampler + Hash3DAnchored + SHShader renderer has {N_RENDERER_STATES}")
    fc, sc = cfg["field"], cfg["shader"]
    log2 = int(fc["log2_table_size"])

    def expect(i, name, dtype, shape, key):
        t = states[i]
        if t.dtype != dtype or (shape is not None and tuple(t.shape) != tuple(shape)):
            want = f"{dtype} {list(shape)}" if shape is not None else str(dtype)
            raise ValueError(f"{path}: state {i} ({name}) is {t.dtype} {list(t.shape)}, {key} expects {want}")

    for i, name, mult in ((0, "tree_nodes", 64), (1, "pers_trans", 544)):
        expect(i, name, torch.uint8, None, "PersSampler")
        if states[i].dim() != 1 or states[i].numel() % mult:
            raise ValueError(f"{path}: state {i} ({name}) must be a 1-D byte blob of whole {mult}-byte records")
    n_nodes, V = states[0].numel() // 64, states[1].numel() // 544
    expect(2, "tree_visit_cnt", torch.int32, (n_nodes,), "PersSampler")
    expect(3, "sub_div_milestones", torch.int32, (states[3].numel(),), "PersSampler")
    expect(4, "feat_pool", torch.float32, ((1 << log2) * N_LEVELS, N_CHANNELS), f"field.log2_table_size = {log2}")
    expect(5, "prim_pool", torch.int32, (N_LEVELS, V, 3), f"the checkpoint's {V} warps")
    expect(6, "bias_pool", torch.float32, (N_LEVELS * V, 3), f"the checkpoint's {V} warps")
    expect(7, "n_volumes", torch.int32, (1,), "Hash3DAnchored")
    if int(states[7].item()) != V:
        raise ValueError(f"{path}: n_volumes {int(states[7].item())} != the checkpoint's {V} warps")
    n_field = _mlp_params(N_LEVELS * N_CHANNELS, int(fc["mlp_hidden_dim"]), int(fc["n_hidden_layers"]))
    expect(8, "field mlp params", torch.float32, (n_field,),
           f"field.mlp_hidden_dim = {fc['mlp_hidden_dim']} / field.n_hidden_layers = {fc['n_hidden_layers']}")
    n_shader = _mlp_params(int(sc["d_in"]), int(sc["d_hidden"]), int(sc["n_hiddens"]))
    expect(9, "shader mlp params", torch.float32, (n_shader,),
           f"shader.d_in = {sc['d_in']} / shader.d_hidden = {sc['d_hidden']} / shader.n_hiddens = {sc['n_hiddens']}")
    expect(10, "app_emb", torch.float32, (n_images, 16),
           f"the image count of dataset.data_path = {cfg['dataset']['data_path']} ({n_images} cameras)")


def check_initial_octree(tree_nodes, pers_trans, cfg, path="renderer.pt"):
    """The rebuilt initial octree (TREE_NODE records) against the checkpoint's warps (``pers_trans`` bytes): one valid leaf
    per warp, and every valid leaf's centre equal, bit for bit, to ``TransInfo.center`` of its ``trans_idx``.  ValueError
    naming the ``pts_sampler`` keys and the data directory the structure was built from otherwise."""
    pc, data = cfg["pts_sampler"], cfg["dataset"]["data_path"]
    built_from = (f"pts_sampler.bbox_levels = {pc['bbox_levels']} / max_level = {pc['max_level']} / split_dist_thres = "
                  f"{pc['split_dist_thres']} over the training cameras of dataset.data_path = {data}")
    trans = np.ascontiguousarray(pers_trans).view(np.uint8).reshape(-1, 544)
    V = trans.shape[0]
    leaves = tree_nodes[tree_nodes["trans_idx"] >= 0]
    if len(leaves) != V:
        raise ValueError(f"{path}: the checkpoint has {V} warps, but the initial octree of {built_from} has {len(leaves)} "
                         "valid leaves")
    want = trans[:, 528:540].copy().view(np.uint32)                              # TransInfo.center
    got = leaves["center"].view(np.uint32)[np.argsort(leaves["trans_idx"])]
    bad = np.nonzero((want != got).any(-1))[0]
    if len(bad):
        raise ValueError(f"{path}: warp {int(bad[0])} is centred at {want[bad[0]].view(np.float32).tolist()}, but the "
                         f"initial octree of {built_from} puts that leaf at {got[bad[0]].view(np.float32).tolist()} "
                         f"({len(bad)} of {V} warps differ)")


def load_scene(config_path, checkpoint_dir=None, device="cuda", trainable=False):
    """A trained scene from the reference's ``runtime_config.yaml`` and a checkpoint directory (default
    ``<base_exp_dir>/checkpoints/latest``) -> ``Scene(global_data_pool, renderer, dataset, iter_step)``.

    Relative paths in the config (``dataset.data_path``, ``base_exp_dir``) are taken against the working directory, as the
    reference program takes them.  Every checkpoint state is checked against the config before anything is built
    (``check_states``); a missing file raises FileNotFoundError.  The sampler is the checkpoint's octree and warps with
    ``pts_sampler.near`` / ``sample_l`` / ``scale_by_dis`` / ``max_oct_intersect_per_ray``; the field keeps the
    checkpoint's primes and biases (no prime draws).  The global data pool is left in VALIDATE mode at the saved iteration's
    ray-march fineness, which is what ``ExpRunner::TestImages`` renders with after training.

    ``trainable=False``: evaluation only.  The checkpoint holds no edge pool, so a TRAIN-mode ``Render`` raises (empty edge
    pool).  ``trainable=True``: what the reference's ``is_continue: true`` resumes with (ExpRunner.cpp:56-58).  The edge pool
    of the initial octree is rebuilt from the training cameras and ``pts_sampler.bbox_levels`` / ``max_level`` /
    ``split_dist_thres`` (``octree_build.initial_octree``), after the rebuilt valid leaves are checked against the checkpoint's
    warps (``check_initial_octree``: ValueError on a count or centre mismatch).  The global data pool also gets the saved
    iteration's gradient-scaling progress.  The scene is still returned in VALIDATE mode; set ``mode_ = TRAIN`` to train."""
    import yaml
    if not os.path.isfile(config_path):
        raise FileNotFoundError(f"load_scene: {config_path} does not exist")
    with open(config_path) as f:
        cfg = yaml.safe_load(f)
    if checkpoint_dir is None:
        checkpoint_dir = os.path.join(cfg["base_exp_dir"], "checkpoints", "latest")
    renderer_pt, scalars_pt = os.path.join(checkpoint_dir, "renderer.pt"), os.path.join(checkpoint_dir, "scalars.pt")
    for p in (renderer_pt, scalars_pt):
        if not os.path.isfile(p):
            raise FileNotFoundError(f"load_scene: {p} does not exist")
    dev = torch.device(device)
    dc, pc, fc, sc, rc, tc = (cfg[k] for k in ("dataset", "pts_sampler", "field", "shader", "renderer", "train"))
    iter_step = load_iter_step(scalars_pt)
    states = load_states(renderer_pt, dev)
    dataset = load_dataset(dc["data_path"], dc["factor"], dc["bounds_factor"], dev)
    check_states(states, cfg, dataset.n_images_, renderer_pt)
    edge_pool = None
    if trainable:
        from .octree_build import initial_octree
        tree_nodes, edge_pool = initial_octree(dataset, pc)
        check_initial_octree(tree_nodes, states[1].cpu().numpy(), cfg, renderer_pt)
        edge_pool = torch.from_numpy(edge_pool.view(np.uint8).reshape(-1))

    gdp = GlobalDataPool()
    sampler = PersSampler(gdp, states[0], states[1], edge_pool, near=float(np.float32(pc["near"])),
                          sample_l=float(np.float32(pc["sample_l"])), scale_by_dis=bool(pc["scale_by_dis"]),
                          max_oct_intersect_per_ray=int(pc["max_oct_intersect_per_ray"]), device=dev)
    field = Hash3DAnchored(gdp, log2_table_size=int(fc["log2_table_size"]), mlp_hidden_dim=int(fc["mlp_hidden_dim"]),
                           mlp_out_dim=int(fc["mlp_out_dim"]), n_hidden_layers=int(fc["n_hidden_layers"]), device=dev,
                           prim_pool=states[5], bias_pool=states[6])
    shader = SHShader(gdp, d_in=int(sc["d_in"]), d_out=int(sc["d_out"]), d_hidden=int(sc["d_hidden"]),
                      n_hiddens=int(sc["n_hiddens"]), degree=int(sc["degree"]), device=dev)
    renderer = Renderer(gdp, sampler, field, shader, n_images=dataset.n_images_, use_app_emb=bool(rc["use_app_emb"]),
                        bg_color=str(rc["bg_color"]), device=dev)
    renderer.LoadStates(states)
    gdp.iter_step_ = iter_step
    gdp.ray_march_fineness_ = ray_march_fineness(iter_step, tc["ray_march_init_fineness"], int(tc["ray_march_fineness_decay_end_iter"]))
    if trainable:
        gdp.gradient_scaling_progress_ = gradient_scaling_progress(iter_step, tc["gradient_scaling_start"],
                                                                   tc["gradient_scaling_end"])
    gdp.mode_ = VALIDATE
    return Scene(gdp, renderer, dataset, iter_step)
