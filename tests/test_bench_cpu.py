"""Host-side logic of bench.py that must not break on the GPU box (no GPU needed): the `config` object both arms print, the clock
sampler on ranks that do not sample, the keys of the committed bench lines."""
import json
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import workloads as W  # noqa: E402


def test_config_object_is_a_pure_function_of_the_flags():
    for cfg in sorted(W.CONFIGS):
        a = bench.config_dict(SimpleNamespace(config=cfg, rays=0), 1)
        b = bench.config_dict(SimpleNamespace(config=cfg, rays=0), 1)
        assert a == b and a["name"] == cfg and "workload" in a and "model" not in a
    strong = bench.config_dict(SimpleNamespace(config="nerf360", rays=0), 8)
    assert strong["rays_per_gpu"] * 8 == strong["global_rays"] == 8192                       # one global batch, split
    weak = bench.config_dict(SimpleNamespace(config="wanjinyou", rays=0), 8)
    assert weak["rays_per_gpu"] == 4096 and weak["global_rays"] == 8 * 4096


def test_clock_sampler_is_inert_on_non_sampling_ranks():
    c = bench.ClockSampler(-1)
    c.poll()
    assert c.rows == [] and "not sampled" in c.err
    s = c.summary()
    assert s["sm_mhz"] is None


def test_committed_bench_lines_carry_the_contract_keys():
    """The bench lines kept under profiles/ (the numbers BASELINE.md quotes) have every key of the bench contract."""
    line = json.loads(open(os.path.join(ROOT, "profiles", "h100_bench.json")).read().strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert k in line, k
    assert line["vs_baseline"] is None and line["roofline"]["bound"] in ("hbm", "tensor") and line["gpu_launches"] > 0
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(line["e2e"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(line["cpu_baseline"])
    ref = json.loads(open(os.path.join(ROOT, "profiles", "h100_bench_ref.json")).read().strip().splitlines()[-1])
    assert ref["impl"] == "reference" and ref["config"] == line["config"] and ref["metric"] == line["metric"]
