"""The bench.py contract on the CPU side: the reference arm (CPU oracle port) prints ONE JSON line with the agreed keys."""
import json
import os
import subprocess
import sys

import helpers as h


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(h.ROOT, "bench.py"), "--impl", "reference", "--points", "3000", "--res", "96",
                          "--sh-degree", "1", "--steps", "2", "--warmup", "1", "--views", "2"],
                         stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "splats/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["steps"] == 2 and d["n_gpus"] == 1 and d["scaling"] == "weak" and d["dtype"] == "f32" and d["data"] == "synthetic"
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "splats/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "model" not in d["config"]


def test_reference_arm_other_ranks_exit_silently():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(h.ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--points", "1000",
                          "--res", "32", "--steps", "1", "--warmup", "1"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                         timeout=300, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_algorithmic_bytes_formula_matches_survey():
    sys.path.insert(0, h.ROOT)
    import bench
    # SURVEY.md §8(d): deg 3 -> 724 B/Gaussian, 52 B/pixel, 44 B/instance; cfg2 = 151.5 MB with N_inst 1.040 M
    assert bench.algorithmic_bytes(1, 16, 0, 0, 0) == 724 and bench.algorithmic_bytes(1, 1, 0, 0, 0) == 184
    assert abs(bench.algorithmic_bytes(100000, 16, 800, 800, 1040000) - 151.44e6) < 0.1e6
