"""The committed bench line (written by `bench.py --gpus 1 --steps 10 --warmup 3` on an H100, card and power limit in README.md)
carries every key the measurement contract names."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(name):
    path = os.path.join(ROOT, "profiles", name)
    if not os.path.exists(path):
        pytest.skip(f"{name} not committed yet")
    with open(path) as f:
        return json.loads(f.read().strip().splitlines()[-1])


def test_single_gpu_line_has_the_contract_keys():
    d = _line("h100_bench_1gpu.json")
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline", "gpu_baseline", "roofline_shading", "step_time_spread"):
        assert k in d, k
    assert d["metric"].startswith("SDS iters/sec") and d["unit"] == "it/s" and d["n_gpus"] == 1 and d["warmup"] >= 3
    assert d["vs_baseline"] is None and d["higher_is_better"] is True and "workload" in d["config"]
    assert abs(d["value"] - 1000.0 / d["ms_per_step"]) < 1e-6 * d["value"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in d["roofline"] and k in d["roofline_kernel"], k
    assert abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-9
    assert d["roofline_kernel"]["traffic"] > 0 and 0 < d["roofline_kernel"]["frac"] <= 1
    # the shader is not HBM-bound: rays/s is reported next to the byte-formula fraction (SURVEY 8d)
    assert d["roofline_shading"]["rays_per_s"] > 1e9 and 0 < d["roofline_shading"]["frac"] < 1
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"], k
    # N1: the condition maps are device-resident; a step ships its camera tensors + ids and reads the loss back
    assert 0 < d["e2e"]["h2d_bytes_per_step"] < 1 << 16 and d["e2e"]["d2h_bytes_per_step"] == 4 and d["e2e"]["value"] != d["value"]
    for k in ("value", "unit", "cores", "kind", "sample", "reps", "sample_seconds"):
        assert k in d["cpu_baseline"], k
    assert d["cpu_baseline"]["kind"] == "port" and d["gpu_launches"] > 500
    assert {"vae_512_fwd_bwd", "shade_128x128_render", "unet_controlnet_3branch_batch_64x64_latents"} <= set(d["cpu_baseline"]["sample_seconds"])
    gb = d["gpu_baseline"]                            # the "same box" bar: stock PyTorch CUDA ops
    assert gb["dense_ms"] > 0 and gb["ours_over_stock"]["dense"] > 1.0
    assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


def test_readme_numbers_are_the_committed_line():
    """The headline table of README.md quotes the committed bench line, not remembered values."""
    readme = open(os.path.join(ROOT, "README.md")).read()
    d = _line("h100_bench_1gpu.json")
    assert f"**{d['value']:.2f}** it/s" in readme and f"{d['e2e']['value']:.2f} it/s" in readme
    assert f"{d['gpu_baseline']['ours_over_stock']['dense']:.2f} x" in readme
