#!/usr/bin/env python
"""Cost of the observation-history width K0 = num_observations x num_observation_history on one GPU, in one process:

  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration with the observation
    set and history length below) at 4096 envs, CUDA events around each iteration from a synchronised device, after warm-up iterations;
  * CUDA-event time of one history roll at 4096 envs over 200 launches with warm L2: go1_history_roll on contiguous 2100-float rows (70
    observations: its float2 kernel), go1_history_roll_pitched on the same rows, and go1_history_roll_pitched at K0 = 2130 (71 x 30,
    2144-float pitch), the roll observe_yaw runs;
  * the card's name and power limit.

    python walk-these-ways_b200/tools/obs_width_bench.py [--envs 4096] [--iters 5] [--warmup 2] [--skip-roll] [--out FILE.json]

K0 % 4 != 0 widths keep their histories at a padded row pitch (go1_b200.capi.history_pitch) so that the first-layer products run on the
tensor cores; --skip-roll times the iterations alone (for a build without go1_history_roll_pitched).
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

# name -> (observe_* flags set on top of scripts/train.py's, num_observations, num_observation_history)
CONFIGS = {
    "70x30": ({}, 70, 30),
    "yaw_71x30": ({"observe_yaw": True}, 71, 30),
    "70x15": ({}, 70, 15),
    "lin_vel_73x31": ({"observe_only_lin_vel": True}, 73, 31),
}


def _cfg(name, envs):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    flags, nobs, hist = CONFIGS[name]
    for k, v in flags.items():
        setattr(Cfg.env, k, v)
    Cfg.env.num_observations, Cfg.env.num_observation_history = nobs, hist
    Cfg.env.num_envs = envs
    return Cfg


def iteration_ms(name, envs, iters, warmup):
    import numpy as np
    import torch
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    Cfg = _cfg(name, envs)
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="obs_width_bench", root=tempfile.mkdtemp(prefix="go1_obs_width_bench_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    _, nobs, hist = CONFIGS[name]
    assert env.num_obs_history == nobs * hist
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
    res = {"K0": nobs * hist, "history_row_pitch": env.obs_history.stride(0), "ms_mean": round(sum(times) / len(times), 2),
           "ms_min": round(min(times), 2), "ms_max": round(max(times), 2)}
    del runner, env
    torch.cuda.empty_cache()
    return res


def roll_us(envs, reps=200, warmup=20):
    import torch
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    out = {}

    def timed(fn):
        for _ in range(warmup):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return round(1000.0 * a.elapsed_time(b) / reps, 2)

    for nobs, hist in ((70, 30), (71, 30)):
        K0 = nobs * hist
        P = capi.history_pitch(K0)
        src, dst = torch.randn(envs, P, device="cuda"), torch.zeros(envs, P, device="cuda")
        obs = torch.randn(envs, nobs, device="cuda")
        if P == K0:
            out[f"roll_{K0}_us"] = timed(lambda: capi.check(L.go1_history_roll(capi.ptr(src), capi.ptr(obs), capi.ptr(dst), envs, nobs, hist, st), "roll"))
        out[f"roll_pitched_{K0}_pitch{P}_us"] = timed(lambda: capi.check(L.go1_history_roll_pitched(capi.ptr(src), P, capi.ptr(obs), capi.ptr(dst), P, envs,
                                                                                                     nobs, hist, st), "roll_pitched"))
        out[f"roll_{K0}_MB_moved"] = round(envs * (2 * K0 + nobs) * 4 / 1e6, 1)     # K0 - nobs read + nobs obs read + K0 written
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--skip-roll", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "obs_width_bench measures on cuda:0 (no CPU fallback)"
    res = {"card": card(), "envs": args.envs, "iterations": {}}
    if not args.skip_roll:
        res["roll"] = roll_us(args.envs)
        print(f"roll: {res['roll']}", file=sys.stderr, flush=True)
    for name in args.configs.split(","):
        res["iterations"][name] = iteration_ms(name, args.envs, args.iters, args.warmup)
        print(f"{name}: {res['iterations'][name]}", file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
