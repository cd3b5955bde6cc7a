"""The reference's own scripts/train.py and scripts/play.py executed unmodified through the drop-in packages
(walk-these-ways_b200/tools/run_reference_scripts.py).  The scripts are reference files and are never committed here: the test
runs where a staging copy exists (`_ref_stage/` or $GO1_REFERENCE_STAGE, made by `run_reference_scripts.py --make-stage`) and is
skipped elsewhere."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE = os.environ.get("GO1_REFERENCE_STAGE", os.path.join(ROOT, "_ref_stage"))


@pytest.mark.skipif(not os.path.exists(os.path.join(STAGE, "scripts", "train.py")), reason="no staged copy of the reference scripts")
def test_reference_train_and_play_scripts_run_unmodified(tmp_path):
    out = tmp_path / "ref.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "walk-these-ways_b200", "tools", "run_reference_scripts.py"), "--stage", STAGE,
                        "--iterations", "2", "--num-envs", "512", "--out", str(out)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    d = json.loads(out.read_text())
    assert d["train"]["iterations_asked_by_script"] == 100000 and d["train"]["weights_finite"] and d["train"]["gemm_impl"] == 1
    assert "ac_weights_last.pt" in d["train"]["checkpoint_files"]
    assert 1.0 < d["play"]["measured_x_vel_mean_last_100"] < 1.9
