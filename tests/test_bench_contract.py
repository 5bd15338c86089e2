"""bench.py's reference arm runs on host cores only, so its JSON line can be checked without a GPU: one line, the keys
a consumer reads, the metric/config of BASELINE.json configs[2] (GenRe full_model inference through the frozen Net.forward,
here on the CPU oracle toolbox + the reference's networks), and the `cpu_baseline` / `e2e` shape.  The arm runs the
reference's own model files, which are not part of this repository: it needs a GenRe-ShapeHD checkout ($GENRE_REF)."""
import json
import os
import subprocess
import sys

import pytest

from conftest import REPO
from genre_shapehd_b200 import compat


@pytest.mark.skipif(compat.find_reference() is None, reason="no GenRe-ShapeHD checkout ($GENRE_REF)")
def test_reference_arm_prints_one_contract_line():
    env = dict(os.environ, RANK="0", WORLD_SIZE="1")
    p = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--cpu-budget", "12"], cwd=REPO, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 1 and d["warmup"] == 0
    assert d["unit"] == "shapes/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["dtype"] == "f32" and d["data"] == "synthetic" and "GenRe" in d["metric"] and "cam_bp" in d["metric"]
    assert "GenRe full_model inference" in d["config"]["workload"] and "configs[2]" in d["config"]["workload"]
    assert d["config"]["batch_per_gpu"] == 16 and d["config"]["voxel_res"] == 128
    shapes_per_step = d["value"] * d["ms_per_step"] * 1e-3               # a whole number of shapes, at most the batch
    assert d["value"] > 0 and 1 <= round(shapes_per_step) <= 16 and abs(shapes_per_step - round(shapes_per_step)) <= 1e-6 * shapes_per_step
    assert d["result_checksum"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1",
                        "--warmup", "0"], cwd=REPO, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip() == ""
