#!/usr/bin/env python
"""Cost of the action FIFO depth L (Cfg.domain_rand.lag_timesteps) on one GPU, in one process:

  * CUDA-event time of one fused env step (go1_step_kernel, mode 0: `decimation` substeps of control + physics + post-physics) at
    4096 envs standing on flat ground, averaged over many launches after warm-up;
  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration) at 4096 envs, CUDA
    events around each iteration from a synchronised device, after warm-up iterations;
  * the card's name and power limit.

    python walk-these-ways_b200/tools/lag_bench.py [--envs 4096] [--iters 5] [--warmup 2] [--out FILE.json]

L = 6 is scripts/train.py's value.  The FIFO moves 96 * L bytes per env and step (12 joints x L slots x 4 B, read once, written once).
"""
import argparse
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

LAGS = (0, 2, 6, 13, 32)


def _cfg(L, envs):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    Cfg.domain_rand.lag_timesteps = L
    Cfg.env.num_envs = envs
    return Cfg


def step_us(L, envs, reps=200, warmup=20):
    import torch
    from go1_b200.config import build_sim_config
    from go1_b200.sim import SimCore
    c, _ = build_sim_config(_cfg(L, envs), num_envs=envs)
    assert c.use_lag == 1 and c.lag_timesteps == L
    sim = SimCore(c)
    sim.env("root_pos")[2].fill_(0.32)
    sim.set_joint_aos("dof_pos", torch.tensor(list(c.default_dof_pos), device="cuda").repeat(envs, 1))
    sim.env("commands")[4].fill_(3.0); sim.env("commands")[8].fill_(0.5)
    actions = torch.randn(envs, 12, device="cuda", generator=torch.Generator("cuda").manual_seed(L)) * 0.3
    for t in range(warmup):
        sim.step(actions, common_step=t, mode=0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for t in range(reps):
        sim.step(actions, common_step=warmup + t, mode=0)
    b.record()
    torch.cuda.synchronize()
    assert torch.isfinite(sim.leg_f32).all()
    sim.close()
    return round(1000.0 * a.elapsed_time(b) / reps, 2)


def iteration_ms(L, envs, iters, warmup):
    import numpy as np
    import torch
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    Cfg = _cfg(L, envs)
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="lag_bench", root=tempfile.mkdtemp(prefix="go1_lag_bench_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    assert env.env.core.cfg.lag_timesteps == L
    runner = Runner(env, device="cuda:0")
    od = env.get_observations()
    state = [od["obs"], od["privileged_obs"], od["obs_history"]]
    times = []
    for it in range(warmup + iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        obs, priv, hist, _ = runner.rollout(*state)
        state = [obs, priv, hist]
        with torch.inference_mode():
            runner.alg.compute_returns(hist[:env.num_train_envs], priv[:env.num_train_envs])
        losses = runner.alg.update()
        b.record()
        torch.cuda.synchronize()
        if it >= warmup:
            times.append(a.elapsed_time(b))
    assert all(np.isfinite(x) for x in losses[:3])
    del runner, env
    torch.cuda.empty_cache()
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "lag_bench measures on cuda:0 (no CPU fallback)"
    res = {"card": card(), "envs": args.envs, "step_kernel_us": {}, "iterations": {}}
    for L in LAGS:
        res["step_kernel_us"][L] = step_us(L, args.envs)
        print(f"L={L}: step {res['step_kernel_us'][L]} us", file=sys.stderr, flush=True)
    for L in LAGS:
        t = iteration_ms(L, args.envs, args.iters, args.warmup)
        res["iterations"][L] = {"ms_mean": round(sum(t) / len(t), 2), "ms_min": round(min(t), 2), "ms_max": round(max(t), 2)}
        print(f"L={L}: {res['iterations'][L]}", file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
