"""bench.py's reference arm on CPU (small graph): the JSON line carries every key the bench contract names,
and only rank 0 prints under a multi-rank launch.  (The GPU arm needs an H100; its line is checked by
running bench.py there.)  Uses oracle/_ref when it is built, else the C restatement -- both are allowed for this arm."""
import json
import os
import subprocess
import sys

from conftest import ROOT

BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "cpu_baseline", "impl"}


def run_bench(extra_env=None):
    env = dict(os.environ)
    env.update(extra_env or {})
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--scale", "12",
                          "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    return out.stdout.strip()


def test_reference_arm_line():
    line = json.loads(run_bench().splitlines()[-1])
    assert BASE_KEYS <= set(line), BASE_KEYS - set(line)
    assert line["impl"] == "reference" and line["n_gpus"] == 1 and line["gpu_launches"] == 0
    assert line["unit"] == "pairs/s" and line["higher_is_better"] is True and line["value"] > 0
    assert "workload" in line["config"] and "model" not in line["config"]
    cb = line["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == line["value"] and cb["sample"]
    assert line["e2e"] == {"value": line["value"], "unit": line["unit"], "h2d_bytes_per_step": 0,
                           "d2h_bytes_per_step": 0}


def test_reference_arm_other_ranks_stay_silent():
    assert run_bench({"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"}) == ""


def test_dump_outputs_files_and_dtypes(tmp_path):
    import numpy as np
    import bench
    lengths = np.array([0, 3, -1, 7], dtype=np.int64)
    valid = np.array([1, 1, 0, 1], dtype=np.uint8)
    bench.dump_outputs(str(tmp_path / "out"), {"lengths": lengths, "valid": valid})
    assert sorted(os.listdir(tmp_path / "out")) == ["lengths.npy", "valid.npy"]
    for name, a in (("lengths", lengths), ("valid", valid)):
        got = np.load(tmp_path / "out" / f"{name}.npy")
        assert got.dtype == np.float64 and np.array_equal(got, a)


def test_dump_outputs_is_refused_by_the_reference_arm(tmp_path):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs",
                          str(tmp_path / "d")], capture_output=True, text=True, timeout=120, cwd=ROOT)
    assert out.returncode != 0 and "--dump-outputs" in out.stderr and not (tmp_path / "d").exists()
