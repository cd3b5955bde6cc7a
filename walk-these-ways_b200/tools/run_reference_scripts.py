#!/usr/bin/env python
"""Executes the REFERENCE's own scripts/train.py and scripts/play.py, unmodified, against the drop-in packages of this
repository (SURVEY.md §8b: "scripts/train.py drops in unchanged").

The scripts are loaded from a staging directory holding verbatim copies of
    <ref>/scripts/train.py, <ref>/scripts/play.py and <ref>/runs/gait-conditioned-agility/pretrain-v0/train/<run>/
        {parameters.pkl, checkpoints/body_latest.jit, checkpoints/adaptation_module_latest.jit}
(`--stage DIR`; `--make-stage --reference <checkout of the reference>` copies them.  The staging directory is git-ignored:
reference files never enter this repository's history).

What is NOT the reference's code here: sys.path (this package + compat/ first), a cap on Runner.learn's iteration count and on
Cfg.env.num_envs (train.py asks for 100000 iterations of 4000 envs), and a recording stand-in for matplotlib (not installed).
"""
import argparse
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time
import types

TOOLS = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(TOOLS)
ROOT = os.path.dirname(PKG)
RUN = "runs/gait-conditioned-agility/pretrain-v0/train"


def make_stage(stage, ref):
    os.makedirs(os.path.join(stage, "scripts"), exist_ok=True)
    for f in ("train.py", "play.py"):
        shutil.copyfile(os.path.join(ref, "scripts", f), os.path.join(stage, "scripts", f))
    run = sorted(os.listdir(os.path.join(ref, RUN)))[0]
    dst = os.path.join(stage, RUN, run, "checkpoints")
    os.makedirs(dst, exist_ok=True)
    shutil.copyfile(os.path.join(ref, RUN, run, "parameters.pkl"), os.path.join(stage, RUN, run, "parameters.pkl"))
    for f in ("body_latest.jit", "adaptation_module_latest.jit"):
        shutil.copyfile(os.path.join(ref, RUN, run, "checkpoints", f), os.path.join(dst, f))
    print("staged", stage)


def load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_train(stage, iterations, num_envs, out):
    import torch
    from ml_logger import logger
    import go1_gym_learn.ppo_cse as ppo_cse
    from go1_gym.envs.go1 import go1_config
    run_root = tempfile.mkdtemp(prefix="go1_reference_scripts_")       # checkpoints are large: keep them out of the tree
    logger.configure(prefix="reference_train_py", root=run_root)
    mod = load(os.path.join(stage, "scripts", "train.py"), "reference_train")
    learn = ppo_cse.Runner.learn
    seen = {}

    def capped(self, num_learning_iterations, **kw):
        seen["asked"] = num_learning_iterations
        seen["num_envs"] = self.env.num_envs
        t0 = time.time()
        learn(self, min(num_learning_iterations, iterations), **kw)
        torch.cuda.synchronize()
        seen["seconds"] = time.time() - t0
        seen["runner"] = self
    ppo_cse.Runner.learn = capped
    config_go1 = go1_config.config_go1

    def config_capped(Cnfg):               # config_go1 sets 4000 envs; everything else is train.py's own configuration
        config_go1(Cnfg)
        Cnfg.env.num_envs = num_envs
    go1_config.config_go1 = config_capped
    try:
        mod.train_go1(headless=True)
    finally:
        ppo_cse.Runner.learn = learn
        go1_config.config_go1 = config_go1
    r = seen["runner"]
    ac = r.alg.actor_critic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    out["train"] = {"iterations_asked_by_script": seen["asked"], "iterations_run": iterations, "num_envs": seen["num_envs"],
                    "seconds": round(seen["seconds"], 2), "gemm_impl": int(AC_Args.gemm_impl), "weights_finite": bool(torch.isfinite(ac.flat_params).all()),
                    "env_steps_per_s": round(iterations * r.num_steps_per_env * seen["num_envs"] / seen["seconds"]),
                    "checkpoint_files": sorted(os.listdir(os.path.join(run_root, "reference_train_py", "checkpoints")))}
    assert out["train"]["weights_finite"]


def run_play(stage, out):
    import numpy as np
    plots = []

    class Ax:
        def plot(self, x, y, *a, **k):
            plots.append((k.get("label"), np.array(y, dtype=np.float64).copy()))

        def __getattr__(self, name):
            return lambda *a, **k: None
    plt = types.ModuleType("matplotlib.pyplot")
    plt.subplots = lambda *a, **k: (None, [Ax(), Ax()])
    plt.tight_layout = lambda *a, **k: None
    plt.show = lambda *a, **k: None
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, plt
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    cwd = os.getcwd()
    os.chdir(os.path.join(stage, "scripts"))          # play.py globs ../runs/<label>/*
    try:
        mod = load(os.path.join(stage, "scripts", "play.py"), "reference_play")
        mod.play_go1(headless=True)
    finally:
        os.chdir(cwd)
    vx = [y for lbl, y in plots if lbl == "Measured" and y.ndim == 1][0]
    out["play"] = {"steps": int(len(vx)), "commanded_x_vel": 1.5, "measured_x_vel_mean_last_100": float(vx[-100:].mean()),
                   "measured_x_vel_min_last_100": float(vx[-100:].min()), "measured_x_vel_first_5": [round(float(v), 3) for v in vx[:5]]}
    assert 1.0 < out["play"]["measured_x_vel_mean_last_100"] < 1.9, out["play"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", default=os.path.join(ROOT, "_ref_stage"))
    ap.add_argument("--make-stage", action="store_true")
    ap.add_argument("--iterations", type=int, default=2)
    ap.add_argument("--num-envs", type=int, default=4096)
    ap.add_argument("--only", default="train,play")
    ap.add_argument("--reference", default=os.environ.get("GO1_REFERENCE_ROOT"), help="--make-stage: a checkout of the reference project")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "go1_reference_scripts.json"))
    a = ap.parse_args()
    if a.make_stage:
        return make_stage(a.stage, a.reference)
    for p in (PKG, os.path.join(PKG, "compat")):
        if p not in sys.path:
            sys.path.insert(0, p)
    out = {"stage": os.path.relpath(a.stage, ROOT)}
    if "train" in a.only:
        run_train(a.stage, a.iterations, a.num_envs, out)
    if "play" in a.only:
        run_play(a.stage, out)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
