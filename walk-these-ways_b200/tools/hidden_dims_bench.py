#!/usr/bin/env python
"""Cost of the AC_Args hidden-layer shapes (actor_hidden_dims = critic_hidden_dims, adaptation_module_branch_hidden_dims) on one GPU, in
one process:

  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration with the shapes below)
    at 4096 envs, CUDA events around each iteration from a synchronised device, after warm-up iterations;
  * CUDA-event time of the fused tails in one forward_all at M = 4096 (a rollout step) and M = 24576 (an update minibatch), from the
    GO1_GEMM_TIMING_CSV dump, with the time of every other tensor-core product of that pass beside it;
  * the card's name and power limit.

    python walk-these-ways_b200/tools/hidden_dims_bench.py [--envs 4096] [--iters 5] [--warmup 2] [--shapes a,b] [--out FILE.json]

A shape the build cannot train reports its error instead of times.
"""
import argparse
import csv
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PKG = os.path.join(ROOT, "walk-these-ways_b200")
for p in (ROOT, PKG, os.path.join(PKG, "compat"), os.path.join(PKG, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from priv_obs_bench import card  # noqa: E402

# name -> (actor / critic hidden dims, adaptation module hidden dims)
SHAPES = {
    "default": ([512, 256, 128], [256, 128]),
    "1024-512-256": ([1024, 512, 256], [512, 256]),
    "256-128-64": ([256, 128, 64], [128, 64]),
    "512-256-128-64": ([512, 256, 128, 64], [256, 128]),
    "500-250-125": ([500, 250, 125], [250, 125]),
}


def _set_shape(name):
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    hidden, adapt = SHAPES[name]
    AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims = list(hidden), list(hidden), list(adapt)


def iteration_ms(name, envs, iters, warmup):
    import numpy as np
    import torch
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    apply_train_config(Cfg)
    Cfg.env.num_envs = envs
    _set_shape(name)
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="hidden_dims_bench", root=tempfile.mkdtemp(prefix="go1_hidden_dims_bench_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    runner = Runner(env, device="cuda:0")
    od = env.get_observations()
    state = [od["obs"], od["privileged_obs"], od["obs_history"]]
    times = []
    for it in range(warmup + iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        obs, priv, h, _ = runner.rollout(*state)
        state = [obs, priv, h]
        with torch.inference_mode():
            runner.alg.compute_returns(h[:env.num_train_envs], priv[:env.num_train_envs])
        losses = runner.alg.update()
        b.record()
        torch.cuda.synchronize()
        if it >= warmup:
            times.append(a.elapsed_time(b))
    assert all(np.isfinite(x) for x in losses[:3])
    res = {"ms_mean": round(sum(times) / len(times), 2), "ms_min": round(min(times), 2), "ms_max": round(max(times), 2)}
    del runner, env
    torch.cuda.empty_cache()
    return res


def forward_us(name, reps=20):
    """Tail launches and the other tensor-core products of one forward_all (mean over `reps` passes after 3 warm ones)."""
    import torch
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse import ActorCritic
    _set_shape(name)
    torch.manual_seed(0)
    NOBS, E, K0, NA = 70, 2, 2100, 12
    ac = ActorCritic(NOBS, E, K0, NA).to("cuda:0")
    ac.flatten()
    out, path = {}, os.path.join(tempfile.mkdtemp(prefix="go1_hidden_dims_bench_"), "gemm.csv")
    os.environ["GO1_GEMM_TIMING_CSV"] = path
    L = capi.lib()
    for M in (4096, 24576):
        h, priv = torch.randn(M, K0, device="cuda") * 0.3, torch.randn(M, E, device="cuda")
        for _ in range(3):
            ac.forward_all(h, priv, tag="bench")
        torch.cuda.synchronize()
        capi.check(L.go1_gemm_timing(1, None, None, None), "timing")
        for _ in range(reps):
            ac.forward_all(h, priv, tag="bench")
        capi.check(L.go1_gemm_timing(0, None, None, None), "timing")
        rows = list(csv.DictReader(open(path)))
        tails = [r for r in rows if r["kernel"].startswith("tail")]
        out[f"M{M}"] = {"tail_launches": len(tails) // reps, "tail_us": round(sum(float(r["us"]) for r in tails) / reps, 1),
                        "other_products": (len(rows) - len(tails)) // reps,
                        "other_products_us": round(sum(float(r["us"]) for r in rows if r not in tails) / reps, 1)}
    del os.environ["GO1_GEMM_TIMING_CSV"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "hidden_dims_bench measures on cuda:0 (no CPU fallback)"
    res = {"card": card(), "envs": args.envs, "shapes": {}}
    for name in args.shapes.split(","):
        r = {"actor_critic_hidden_dims": SHAPES[name][0], "adaptation_hidden_dims": SHAPES[name][1]}
        try:
            r["forward_all"] = forward_us(name)
            r["iteration"] = iteration_ms(name, args.envs, args.iters, args.warmup)
        except Exception as e:      # the shape does not train on this build: say so
            r["error"] = f"{type(e).__name__}: {e}"[:300]
        res["shapes"][name] = r
        print(f"{name}: {r}", file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
