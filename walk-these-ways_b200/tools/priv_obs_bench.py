#!/usr/bin/env python
"""Cost of the privileged-observation width E (num_privileged_obs) on one GPU, in one process:

  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration) at 4096 envs for
    E = 2 (train.py: friction + restitution), 5 (+ body velocity), 18 and 45 (every priv_observe_* group), CUDA events around each
    iteration from a synchronised device, after warm-up iterations;
  * CUDA-event times of the trailing-input kernels at the shapes of that run (go1_mlp_extra_forward on the rollout and minibatch rows,
    go1_mlp_extra_backward: d(latent) from the transposed first-layer dz, and the row-major pass with the weight gradient);
  * the card's name and power limit.

    python walk-these-ways_b200/tools/priv_obs_bench.py [--envs 4096] [--iters 5] [--warmup 2] [--out FILE.json]

E <= 4 rides in the GEMM epilogues (no trailing-input kernel runs in training); E > 4 runs the wide kernels.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PKG = os.path.join(ROOT, "walk-these-ways_b200")
for p in (ROOT, PKG, os.path.join(PKG, "compat")):
    if p not in sys.path:
        sys.path.insert(0, p)

WIDTHS = {"friction": 1, "restitution": 1, "base_mass": 1, "com_displacement": 3, "motor_strength": 12, "motor_offset": 12, "body_height": 1,
          "body_velocity": 3, "gravity": 3, "clock_inputs": 4, "desired_contact_states": 4}
GROUPS = {
    2: ("friction", "restitution"),
    5: ("friction", "restitution", "body_velocity"),
    18: ("friction", "restitution", "body_velocity", "motor_strength", "base_mass"),
    45: tuple(WIDTHS),
}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        limit = q.stdout.strip()
    except Exception as e:      # the timing stands without it; say so instead of guessing
        limit = f"unavailable ({type(e).__name__})"
    return {"name": name, "power_limit_and_max_sm_clock": limit}


def iteration_ms(E, envs, iters, warmup):
    import numpy as np
    import torch
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    apply_train_config(Cfg)
    for name in WIDTHS:
        setattr(Cfg.env, "priv_observe_" + name, name in GROUPS[E])
    Cfg.env.num_privileged_obs = E
    Cfg.env.num_envs = envs
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="priv_obs_bench", root=tempfile.mkdtemp(prefix="go1_priv_obs_bench_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    assert env.num_privileged_obs == E
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


def kernel_us(E, M_roll, M_mb, reps=50):
    """Per-call times of the trailing-input kernels for E at the default layer widths (o = 512)."""
    import torch
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    o, K0 = 512, 2100
    W = torch.randn(o, K0 + E, device="cuda") * 0.02
    w = W[:, K0:]
    out = {}

    def timed(fn):
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return round(1000.0 * a.elapsed_time(b) / reps, 2)

    for M in (M_roll, M_mb):
        y, ex = torch.randn(M, 1280, device="cuda")[:, 768:], torch.randn(M, E, device="cuda")
        act = capi.act_arg(capi.ACTIVATIONS["elu"], 1)
        out[f"extra_forward_M{M}"] = timed(lambda: capi.check(L.go1_mlp_extra_forward(capi.ptr(y), y.stride(0), capi.ptr(ex), E, capi.ptr(w), K0 + E, M, o, E, act, st), "fwd"))
    M = M_mb
    ex, dx = torch.randn(M, E, device="cuda"), torch.empty(M, E, device="cuda")
    dzT = torch.randn(o, (M + 31) // 32 * 32, device="cuda")
    dz = torch.randn(M, o, device="cuda")
    g = torch.empty(o, K0 + E, device="cuda")
    out[f"extra_backward_dextra_transposed_M{M}"] = timed(lambda: capi.check(L.go1_mlp_extra_backward(
        capi.ptr(dzT), dzT.stride(0), 1, None, 0, capi.ptr(w), K0 + E, None, 0, capi.ptr(dx), E, M, o, E, 0, st), "bwd"))
    out[f"extra_backward_dextra_and_wgrad_M{M}"] = timed(lambda: capi.check(L.go1_mlp_extra_backward(
        capi.ptr(dz), o, 0, capi.ptr(ex), E, capi.ptr(w), K0 + E, capi.ptr(g[:, K0:]), K0 + E, capi.ptr(dx), E, M, o, E, 0, st), "bwd"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "priv_obs_bench measures on cuda:0 (no CPU fallback)"
    res = {"card": card(), "envs": args.envs, "iterations": {}, "kernels_us": {}}
    M_mb = args.envs * 24 // 4
    for E in GROUPS:
        t = iteration_ms(E, args.envs, args.iters, args.warmup)
        res["iterations"][E] = {"ms_mean": round(sum(t) / len(t), 2), "ms_min": round(min(t), 2), "ms_max": round(max(t), 2)}
        print(f"E={E}: {res['iterations'][E]}", file=sys.stderr, flush=True)
        if E > 4:
            res["kernels_us"][E] = kernel_us(E, args.envs, M_mb)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
