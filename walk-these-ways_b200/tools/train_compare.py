#!/usr/bin/env python
"""Learning-level evidence for the TF32 path (VERDICT r1, weak #2): trains scripts/train.py's configuration for K iterations
with the tcgen05 TF32 GEMMs (AC_Args.gemm_impl = 1) and with the exact-fp32 CUDA-core GEMMs (impl 0) -- or, with --impls 1,2, the
BF16 history products (impl 2), or with 2b impl 2 plus AC_Args.bf16_backward -- from the same seeds and
writes the reward-term trajectories (one record per `log_freq` iterations, like the reference's metrics.pkl) next to the first
records of the shipped training log (tests/golden/metrics_envelope.json: Isaac Gym, 4000 envs).
    python walk-these-ways_b200/tools/train_compare.py --iterations 200 --out train_compare.json"""
import argparse
import json
import os
import tempfile
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import torch  # noqa: E402

KEYS = ["train/episode/rew_total/mean", "train/episode/rew_tracking_lin_vel/mean", "train/episode/rew_tracking_ang_vel/mean",
        "train/episode/rew_tracking_contacts_shaped_force/mean", "train/episode/rew_tracking_contacts_shaped_vel/mean",
        "train/episode/rew_collision/mean", "train/episode/rew_action_rate/mean", "train/episode/rew_torques/mean",
        "train/episode/command_area_trot/mean", "adaptation_loss/mean", "mean_value_loss/mean", "mean_surrogate_loss/mean", "iterations"]


NAMES = {"0": "fp32", "1": "tf32", "2": "bf16", "2b": "bf16_backward"}


def run(impl, iterations, envs, tag, bf16_backward=False):
    import numpy as np
    from ml_logger import logger
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.bf16_backward = bf16_backward
    torch.manual_seed(0); np.random.seed(0)
    env, runner = bench.build_training(envs, "cuda:0", impl, "flat")
    from go1_gym_learn.ppo_cse import RunnerArgs
    RunnerArgs.log_freq, RunnerArgs.save_interval, RunnerArgs.save_video_interval = 10, 10 ** 9, 0
    logger.configure(prefix=f"train_compare_{tag}", root=tempfile.mkdtemp(prefix="go1_train_compare_"))
    logger.summaries = []
    t0 = time.time()
    runner.learn(num_learning_iterations=iterations, init_at_random_ep_len=True, eval_freq=100)
    torch.cuda.synchronize()
    dt = time.time() - t0
    rows = list(logger.summaries)
    out = {k: [r.get(k) for r in rows] for k in KEYS}
    out["seconds"] = round(dt, 1)
    out["env_steps_per_s_incl_logging"] = round(iterations * 24 * envs / dt)
    del env, runner
    torch.cuda.empty_cache()
    AC_Args.bf16_backward = False
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=200)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--impls", default="1,0", help="comma-separated AC_Args.gemm_impl values: 0 fp32, 1 tf32, 2 bf16; 2b = 2 with AC_Args.bf16_backward")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "go1_train_compare.json"))
    a = ap.parse_args()
    res = {"iterations": a.iterations, "envs": a.envs}
    for m in a.impls.split(","):
        res[NAMES[m]] = run(int(m.rstrip("b")), a.iterations, a.envs, f"impl{m}", bf16_backward=m.endswith("b"))
    with open(os.path.join(ROOT, "tests", "golden", "metrics_envelope.json")) as f:
        env = json.load(f)
    n = a.iterations // 10 + 1
    res["reference_isaacgym_4000_envs"] = {k: v[:n] for k, v in env.items()}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f)
    for name in ("tf32", "fp32", "bf16", "bf16_backward", "reference_isaacgym_4000_envs"):
        if name in res:
            r = res[name]
            print(name, "rew_total", [None if x is None else round(x, 3) for x in r["train/episode/rew_total/mean"][::4]],
                  "tracking_lin_vel", [None if x is None else round(x, 4) for x in r["train/episode/rew_tracking_lin_vel/mean"][::4]])
