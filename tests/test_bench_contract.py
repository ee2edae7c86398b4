"""CPU: the bench.py JSON contract of the reference arm (the CPU-oracle timing itself is stubbed: it takes a minute per sample)
and the synthetic workload definitions of the four BASELINE configs."""
import json
import sys
import types


def test_reference_arm_line(monkeypatch, capsys):
    sys.path.insert(0, ".")
    import bench
    monkeypatch.setattr(bench, "cpu_oracle_seconds_per_image", lambda cfg, verbose=False: (200.0, 32, "stub sample"))
    args = types.SimpleNamespace(gpus=1, steps=2, warmup=1, ref_budget_s=1e9)
    monkeypatch.delenv("RANK", raising=False)
    bench.run_reference(args, bench.CONFIGS[1])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "images/s" and line["higher_is_better"] is True
    assert abs(line["value"] - 1 / 200.0) < 1e-12 and line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] == 32
    assert line["e2e"] == {"value": line["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["metric"] == bench.METRIC and line["gpu_launches"] == 0
    assert line["steps"] == 2 and line["warmup"] == 1          # the number of samples actually timed


def test_reference_arm_reports_the_samples_it_timed(monkeypatch, capsys):
    """a wall-clock budget that allows one sample only: `steps` must say 1, not the requested 20"""
    sys.path.insert(0, ".")
    import bench
    t = {"now": 0.0}
    monkeypatch.setattr(bench.time, "perf_counter", lambda: t["now"])

    def fake(cfg, verbose=False):
        t["now"] += 100.0
        return 100.0, 32, "stub"
    monkeypatch.setattr(bench, "cpu_oracle_seconds_per_image", fake)
    monkeypatch.delenv("RANK", raising=False)
    bench.run_reference(types.SimpleNamespace(gpus=1, steps=20, warmup=5, ref_budget_s=240.0), bench.CONFIGS[1])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line["steps"] == 1 and line["warmup"] == 1, (line["steps"], line["warmup"])


def test_reference_arm_other_ranks_are_silent(monkeypatch, capsys):
    sys.path.insert(0, ".")
    import bench
    monkeypatch.setenv("RANK", "1")
    bench.run_reference(types.SimpleNamespace(gpus=2, steps=1, warmup=0, ref_budget_s=1.0), bench.CONFIGS[1])
    assert capsys.readouterr().out == ""


def test_config_workloads():
    sys.path.insert(0, ".")
    import bench
    assert sorted(bench.CONFIGS) == [1, 2, 3, 4]
    for c, cfg in bench.CONFIGS.items():
        ids, am, pos_map, is_thing = bench.batch_text(cfg, cfg["batch"])
        assert ids.shape == (cfg["batch"], cfg["lt"]) and am.shape == ids.shape
        if cfg["task"] == "grounding":
            assert pos_map == {1: [0]} and not bool((ids[0] == ids[1]).all())      # one expression per image
        else:
            assert len(pos_map) == cfg["classes"] and bool((ids[0] == ids[1]).all())
            assert max(max(v) for v in pos_map.values()) < int(am[0].sum())
    assert int(bench.batch_text(bench.CONFIGS[4], 1)[1].sum()) > 512             # ADE-847 prompt takes the BERT chunk path


def test_committed_product_line_follows_the_contract():
    """The bench line committed under profiles/ (one H100, config 1) carries every key of the bench contract plus the roofline /
    cpu_baseline objects, and its derived numbers are consistent with each other."""
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    need = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
            "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"}
    line = json.loads(open(os.path.join(root, "profiles", "h100_bench_config1.json")).read())
    assert need <= set(line), need - set(line)
    assert line["n_gpus"] == 1 and line["unit"] == "images/s" and line["scaling"] == "weak" and line["vs_baseline"] is None
    B = line["config"]["per_gpu_batch"]
    assert abs(line["value"] - B / (line["ms_per_step"] / 1000.0)) < 1e-6 * line["value"]
    assert line["e2e"]["h2d_bytes_per_step"] > 0 and line["e2e"]["d2h_bytes_per_step"] > 0 and line["e2e"]["value"] < line["value"]
    assert line["gpu_launches"] > 500 * line["steps"]          # ~1000 library kernels per captured step
    r = line["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic", "kernels", "gemm_tc_all", "vit_h_forward_alone"} <= set(r)
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and 0.0 < r["frac"] < 1.0
    top = r["kernels"][r["kernel"]]
    assert top["share_of_timed_kernels"] == max(k["share_of_timed_kernels"] for k in r["kernels"].values())
    assert r["mma_passes"] == top["mma_pass_equivalents"] and abs(r["executed_frac"] - r["frac"] * r["mma_passes"]) < 1e-9
    assert not set(line["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    cpu = line["cpu_baseline"]
    assert cpu["kind"] == "port" and cpu["cores"] >= 1 and cpu["value"] > 0 and "sample" in cpu
    assert 0.0 < r["vit_h_forward_alone"]["frac"] < 1.0
