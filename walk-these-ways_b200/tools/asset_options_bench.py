#!/usr/bin/env python
"""Cost of the asset options (Cfg.asset, go1_sim_set_asset_options, DESIGN.md §3) at their Go1 defaults, against a parent build:

  * the step kernel alone (go1_step_kernel, mode 0: 4 substeps + post-physics): its device time per launch from torch.profiler, and
    the CUDA-event time of the whole env step (go1_step_kernel + go1_event_fill_kernel, as sim.step launches them), at 4096 and
    65536 envs standing on flat ground under random actions, with a 512 MiB L2 flush before every launch (as
    tools/self_collision_bench.py);
  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration) at 4096 envs,
    CUDA events around each iteration from a synchronised device;
  * the card's name and power limit.

Each round runs one worker process per build, the order alternating from round to round; a worker imports the package of its
tree.  The parent tree is a checkout of the parent commit's walk-these-ways_b200/ and include/ with its library built, e.g.

    mkdir -p build/parent && git archive <parent> walk-these-ways_b200 include | tar -x -C build/parent
    make -C build/parent/walk-these-ways_b200/csrc
    python walk-these-ways_b200/tools/asset_options_bench.py --parent build/parent [--rounds 5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _paths(tree):
    pkg = os.path.join(tree, "walk-these-ways_b200")
    return [pkg, os.path.join(pkg, "compat"), os.path.join(pkg, "tools")]


def _cfg(envs):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    Cfg.env.num_envs = envs
    return Cfg


def step_ms(envs, reps=40, warmup=5):
    import torch
    from go1_b200.config import build_sim_config
    from go1_b200.sim import SimCore
    c, info = build_sim_config(_cfg(envs), num_envs=envs)
    sim = SimCore(c, self_collision=info["self_collision"])      # the asset options stay at go1_sim_create's Go1 defaults
    sim.env("root_pos")[2].fill_(0.32)
    sim.set_joint_aos("dof_pos", torch.tensor(list(c.default_dof_pos), device="cuda").repeat(envs, 1))
    sim.env("commands")[4].fill_(3.0); sim.env("commands")[8].fill_(0.5)
    actions = torch.randn(envs, 12, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 0.3
    flush = torch.empty(512 * 1024 * 1024 // 4, device="cuda")
    times = []
    for t in range(warmup + reps):
        flush.fill_(float(t))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sim.step(actions, common_step=t, mode=0)
        b.record()
        torch.cuda.synchronize()
        if t >= warmup:
            times.append(a.elapsed_time(b))
    # the step kernel alone: device time of every go1_step_kernel launch, from the profiler's kernel records (a run of its own)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(reps):
            flush.fill_(float(t))
            sim.step(actions, common_step=warmup + reps + t, mode=0)
        torch.cuda.synchronize()
    kern = sorted(e.time_range.elapsed_us() / 1000.0 for e in prof.events()
                  if e.device_type == torch.autograd.DeviceType.CUDA and "go1_step_kernel" in e.name)
    assert len(kern) == reps, len(kern)
    assert torch.isfinite(sim.leg_f32).all()
    state = torch.cat([sim.env_f32.flatten(), sim.leg_f32.flatten(), sim.obs.flatten(), sim.rew]).double()
    sim.close()
    del flush
    torch.cuda.empty_cache()
    return sorted(times)[len(times) // 2], kern[len(kern) // 2], float(state.sum()), float(state.abs().sum())


def iteration_ms(envs, iters, warmup):
    import numpy as np
    import torch
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    Cfg = _cfg(envs)
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="asset_options_bench", root=tempfile.mkdtemp(prefix="go1_asset_options_bench_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
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
    return times


def worker(args):
    sys.path[:0] = _paths(args.tree)
    from go1_b200 import capi
    assert os.path.dirname(os.path.dirname(capi.LIB_PATH)) == os.path.join(os.path.abspath(args.tree), "walk-these-ways_b200"), capi.LIB_PATH
    res = {"step_ms": {}, "kernel_ms": {}, "step_checksum": {}}
    for envs in (4096, 65536):
        ms, kms, s, sa = step_ms(envs)
        res["step_ms"][envs] = ms
        res["kernel_ms"][envs] = kms
        res["step_checksum"][envs] = [s, sa]
    res["iteration_ms"] = iteration_ms(4096, args.iters, args.warmup)
    print("RESULT " + json.dumps(res), flush=True)


def _run(tree, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--tree", tree, "--iters", str(args.iters), "--warmup", str(args.warmup)]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=tempfile.gettempdir())
    line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
    if p.returncode != 0 or not line:
        raise RuntimeError(f"worker for {tree} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    return json.loads(line[-1][7:])


def _stats(v, nd):
    v = sorted(v)
    return {"median": round(v[len(v) // 2], nd), "min": round(v[0], nd), "max": round(v[-1], nd), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent build (walk-these-ways_b200/ with its lib/, include/)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    import torch
    assert torch.cuda.is_available(), "asset_options_bench measures on cuda:0 (no CPU fallback)"
    sys.path[:0] = _paths(ROOT)
    from priv_obs_bench import card
    trees = {"this": ROOT}
    if args.parent:
        trees["parent"] = os.path.abspath(args.parent)
    runs = {k: [] for k in trees}
    for r in range(args.rounds):
        order = list(trees) if r % 2 == 0 else list(reversed(trees))
        for k in order:
            runs[k].append(_run(trees[k], args))
            print(f"round {r} {k}: kernel {runs[k][-1]['kernel_ms']} step {runs[k][-1]['step_ms']} iteration {[round(x, 1) for x in runs[k][-1]['iteration_ms']]}", file=sys.stderr, flush=True)
    res = {"card": card(), "rounds": args.rounds, "step_kernel_ms": {}, "env_step_ms": {}, "iteration_ms": {}, "same_results": None}
    for envs in ("4096", "65536"):
        res["step_kernel_ms"][envs] = {k: _stats([x["kernel_ms"][envs] for x in v], 4) for k, v in runs.items()}
        res["env_step_ms"][envs] = {k: _stats([x["step_ms"][envs] for x in v], 4) for k, v in runs.items()}
    res["iteration_ms"] = {k: _stats([t for x in v for t in x["iteration_ms"]], 2) for k, v in runs.items()}
    if "parent" in runs:       # the default options compute what the parent computed: the step checksums agree bit for bit
        res["same_results"] = all(x["step_checksum"] == y["step_checksum"] for x, y in zip(runs["this"], runs["parent"]))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
