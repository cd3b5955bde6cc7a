#!/usr/bin/env python
"""bench.py — Go1 env-steps/s at 4096 envs per GPU (BASELINE.json metric), one JSON line on rank 0.

A "step" is one training iteration of scripts/train.py's configuration, always from the same seeded state: a 24-step rollout of 4096 envs
(policy inference + fused sim step + device-resident command curriculum, one CUDA graph replay per env step)
followed by compute_returns and the full PPO update (5 epochs x 4 minibatches + adaptation steps).
value = env-steps of all ranks / device time (CUDA events, max over ranks); e2e = the same through the public
API by host wall clock, including every host<->device copy of the path (with the device curriculum: the
read-back of the loss scalars, 28 bytes per iteration -- nothing else of this on-device RL loop crosses PCIe).

    python bench.py --gpus 1 --steps 3 --warmup 3
    python -m torch.distributed.run --nproc-per-node N ... bench.py --gpus N ...
    python bench.py --impl reference        # the CPU port of the reference path on the host cores
    python bench.py --dump-outputs DIR      # after the timed steps: what the last one returned, as DIR/<name>.npy

Nothing is written next to this file: run logs, profiles and dumps go to a temporary directory or to the directory named.

Workloads (BASELINE.json `configs`):  --config flat (default; configs[1]: scripts/train.py, 4096 envs per GPU, weak scaling)
  --config rough_dr   configs[2]: rough height field + full domain randomisation incl. pushes, 4096 envs in total, strong-sharded
  --config mob16k     configs[3]: scripts/train.py's gait-conditioned (MoB) command curriculum, 16384 envs in total, strong-sharded
  --config sweep      configs[4]: env-count sweep 1k..128k per GPU: sim-step env-steps/s + GB/s, and whole-iteration env-steps/s
  --scaling weak|strong overrides the default of the config; --envs = envs per GPU (weak) or in total (strong).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "walk-these-ways_b200")
for p in (ROOT, PKG, os.path.join(PKG, "compat"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

METRIC = "env_steps_per_s"
UNIT = "env-steps/s"
T_ROLLOUT = 24

# fp32 words the fused step kernel reads / writes per env-step in its SoA layout (DESIGN.md §4): every row it
# touches, counted once.  reads: root 13, q/qd 24, motor_offsets 12, actions 12, DR 9, prev foot vel 12, action FIFO 72,
# actuator lags 48, ep_len 1, commands 15, gait 1, last_* 60, last_contacts 4, episode/command sums (RMW) 44
# writes: FIFO 72, lags 48, torques+target 24, q/qd 24, root 13, foot pos/vel/prev 36, contact forces 60, gait outputs 20,
# base-frame 9, actions 12, gait 1, rew pos/neg 2, rew/reset/timeout/ep_len 4, obs 70, priv 2, last_* 60, sums 44, contacts 4
SIM_READ_WORDS = 13 + 24 + 12 + 12 + 9 + 12 + 72 + 48 + 1 + 15 + 1 + 60 + 4 + 44
SIM_WRITE_WORDS = 72 + 48 + 24 + 24 + 13 + 36 + 60 + 20 + 9 + 12 + 1 + 2 + 4 + 70 + 2 + 60 + 44 + 4
SIM_BYTES_PER_ENV_STEP = 4 * (SIM_READ_WORDS + SIM_WRITE_WORDS)


def peaks():
    """(HBM GB/s, dense TF32 TFLOP/s, source): the H100 SXM data-sheet figures (HBM3 3.35 TB/s, 495 TFLOP/s dense TF32 at a 700 W
    limit) -- ceilings for the share-of-peak fields, not rates this program reached."""
    return 3350.0, 495.0, "H100 SXM data sheet"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index=0):
        self.lines, self.proc, self.idx = [], None, gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "200", "-i", str(self.idx)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for l in self.lines:
            f = [x.strip() for x in l.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons), "samples": len(sm)}


ROUGH_DR_OVERRIDES = {
    # BASELINE.json configs[2] / SURVEY.md §8(d) config 3: rough height field (default terrain_proportions, 10 x 20 tiles of 8 m) and
    # the full domain randomisation of legged_robot_config.py (friction, restitution, mass, com, motor strength / offset, Kp / Kd,
    # gravity, pushes, lag), re-drawn at resets and every rand_interval (randomize_rigids_after_start)
    "terrain": dict(mesh_type="heightfield", terrain_proportions=[0.1, 0.1, 0.35, 0.25, 0.2], num_rows=10, num_cols=20, terrain_length=8.0,
                    terrain_width=8.0, horizontal_scale=0.1, vertical_scale=0.005, border_size=25.0, curriculum=True, center_robots=False,
                    teleport_robots=True, teleport_thresh=2.0, terrain_noise_magnitude=0.1, x_init_range=1.0, y_init_range=1.0),
    "domain_rand": dict(randomize_rigids_after_start=True, randomize_com_displacement=True, randomize_Kp_factor=True, randomize_Kd_factor=True,
                        push_robots=True, push_interval_s=15, max_push_vel_xy=1.0),
}
CONFIGS = {
    "flat": dict(workload="Go1 flat terrain, 4096 envs/GPU, 24-step rollout + ppo_cse update (scripts/train.py config)", envs=4096, scaling="weak"),
    "rough_dr": dict(workload="Go1 rough height field + full domain randomisation (pushes, rigid/motor re-randomisation, gravity), 4096 envs total, "
                              "24-step rollout + ppo_cse update", envs=4096, scaling="strong"),
    "mob16k": dict(workload="Go1 gait-conditioned MoB command curriculum (scripts/train.py config), 16384 envs total, 24-step rollout + ppo_cse update",
                   envs=16384, scaling="strong"),
    "sweep": dict(workload="Go1 flat terrain env-count sweep (per GPU): fused sim step alone, and 24-step rollout + ppo_cse update", envs=4096, scaling="weak"),
}


def resolve_envs(args, world):
    spec = CONFIGS[args.config]
    scaling = args.scaling or spec["scaling"]
    n = args.envs if args.envs else spec["envs"]
    if scaling == "strong":
        assert n % world == 0, "strong scaling: the env count must divide by the number of GPUs"
        n //= world
    return scaling, n


def config_dict(args, world, envs_per_gpu):
    """The workload definition both arms print (the reference arm times a bounded sample of it, named in its cpu_baseline)."""
    return {"workload": CONFIGS[args.config]["workload"], "name": args.config, "envs_per_gpu": envs_per_gpu, "envs_total": envs_per_gpu * world,
            "rollout_steps": T_ROLLOUT, "parallelism": f"dp{world}",
            "l2_policy": "iteration and GEMM timing use the live working set (rollout slab 0.87 GB and minibatch operands 0.2 GB > L2); "
                         "the sim-step kernel is timed alone with a 512 MiB L2 flush between launches",
            "gemm_impl": "fp32 CUDA cores" if args.gemm == 0 else "wgmma tf32"}


def build_training(num_envs, device, gemm_impl, config="flat"):
    import numpy as np
    import torch
    import importlib
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]                 # a fresh Cfg tree per build (the sweep builds several envs in one process)
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    from ml_logger import logger
    torch.manual_seed(0)                   # same arguments -> same initial weights, env state and action noise from run to run
    np.random.seed(0)
    apply_train_config(Cfg)
    if config == "rough_dr":
        for sec, kv in ROUGH_DR_OVERRIDES.items():
            for k, v in kv.items():
                setattr(getattr(Cfg, sec), k, v)
        np.random.seed(0)                  # terrain generator stream
    Cfg.env.num_envs = num_envs
    AC_Args.gemm_impl = gemm_impl
    RunnerArgs.num_steps_per_env = T_ROLLOUT
    logger.configure(prefix="bench", root=tempfile.mkdtemp(prefix="go1_bench_runs_"))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device=device, headless=True, cfg=Cfg))
    runner = Runner(env, device=device)
    env.episode_length_buf = torch.randint_like(env.episode_length_buf, high=int(env.max_episode_length))   # learn(init_at_random_ep_len=True)
    return env, runner


class StateSnapshot:
    """Everything mutable that a training iteration reads, reachable from the given roots: the bytes of every tensor storage, numpy array
    and ctypes structure, numpy RandomState streams, and the scalar attributes of every object on the way (the membership of lists and dicts -- caches of
    captured graphs and packed operands -- is left as it is).  restore() puts it all back
    IN PLACE (captured CUDA graphs and the library keep their pointers).  Storages beyond SKIP_BYTES are left alone: those are the
    rollout slab and the minibatch operands, which an iteration rewrites in full before it reads them."""
    SKIP_BYTES = 128 * 1024 * 1024
    COUNTERS = ("h2d_bytes", "d2h_bytes", "iters_counted")      # what bench.py itself counts over the timed window

    def __init__(self, roots):
        import ctypes
        import types
        import numpy as np
        import torch
        self.torch, self.np, self.ctypes = torch, np, ctypes
        self.storages, self.arrays, self.structs, self.rngs, self.scalars = {}, [], [], [], []
        seen, stack = set(), list(roots)
        leaf = (str, bytes, int, float, bool, type(None))
        skip = (types.ModuleType, types.FunctionType, types.MethodType, types.BuiltinFunctionType, type, torch.cuda.CUDAGraph, torch.cuda.Stream,
                torch.cuda.Event, torch.Generator, torch.device, torch.dtype)
        while stack:
            o = stack.pop()
            if isinstance(o, leaf) or isinstance(o, skip) or id(o) in seen:
                continue
            seen.add(id(o))
            if isinstance(o, torch.Tensor):
                st = o.untyped_storage()
                if st.data_ptr() and st.data_ptr() not in self.storages and 0 < st.nbytes() <= self.SKIP_BYTES:
                    flat = torch.empty(0, dtype=torch.uint8, device=o.device).set_(st)
                    self.storages[st.data_ptr()] = (flat, flat.clone())
                continue
            if isinstance(o, np.ndarray):
                if o.dtype != object and o.flags.writeable:
                    self.arrays.append((o, o.copy()))
                continue
            if isinstance(o, np.random.RandomState):
                self.rngs.append((o, o.get_state()))
                continue
            if isinstance(o, (ctypes.Structure, ctypes.Array)):
                self.structs.append((o, bytes(o)))
                continue
            if isinstance(o, dict):
                stack.extend(o.values())
                continue
            if isinstance(o, (list, tuple, set, frozenset)):
                stack.extend(o)
                continue
            d = getattr(o, "__dict__", None)
            if isinstance(d, dict):
                self.scalars.append((o, {k: v for k, v in d.items() if k not in self.COUNTERS and
                                         (isinstance(v, leaf) or (isinstance(v, tuple) and all(isinstance(x, leaf) for x in v)))}))
                stack.extend(d.values())
        self.np_global = np.random.get_state()
        self.torch_cpu, self.torch_cuda = torch.get_rng_state(), torch.cuda.get_rng_state()

    def restore(self):
        for flat, saved in self.storages.values():
            flat.copy_(saved)
        for a, saved in self.arrays:
            a[...] = saved
        for o, raw in self.structs:
            self.ctypes.memmove(self.ctypes.addressof(o), raw, len(raw))
        for r, st in self.rngs:
            r.set_state(st)
        for o, kv in self.scalars:
            for k, v in kv.items():
                try:
                    setattr(o, k, v)
                except Exception:
                    pass
        self.np.random.set_state(self.np_global)
        self.torch.set_rng_state(self.torch_cpu)
        self.torch.cuda.set_rng_state(self.torch_cuda)


def run_b200(args):
    import torch
    import torch.distributed as dist
    from go1_b200 import capi
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the GPU path has no CPU fallback; use --impl reference for the CPU port)")
    torch.cuda.set_device(local)
    device = f"cuda:{local}"
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(device))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torchrun for N>1"
    scaling, envs_per_gpu = resolve_envs(args, world)
    if args.config == "sweep":
        return run_sweep(args, world, rank, local, device)
    env, runner = build_training(envs_per_gpu, device, args.gemm, args.config)
    L = capi.lib()
    od = env.get_observations()
    state0 = [od["obs"], od["privileged_obs"], od["obs_history"]]
    state = list(state0)
    # Every iteration, warm-up or timed, starts from the seeded state (weights, optimizer moments, learning rate, env and curriculum
    # state, counters of the random streams), put back in place before it runs, so that a run is reproducible from its arguments
    # (the first iteration, which captures the CUDA graphs, still differs from the later ones; compare runs with equal --steps / --warmup): the closed loop of policy, contact physics and Adam turns
    # last-bit differences of the atomically accumulated gradients into different trajectories within a few iterations, and then neither
    # two runs nor two builds could be compared output for output.  Putting the state back is not part of the timed step: every iteration is
    # timed on its own (CUDA events and host clock from a synchronised device to a synchronised device) and the timed ones are summed.
    snap = StateSnapshot([env, runner, state0])

    phase_ms = [0.0, 0.0, 0.0, 0]
    spent = [0.0, 0.0]                     # device ms, host seconds of the iterations run so far

    def iteration():
        snap.restore()
        state[:] = state0
        ea, eb = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        tw = time.perf_counter()
        ea.record()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if args.breakdown else None
        if ev: ev[0].record()
        obs, priv, hist, infos = runner.rollout(*state)
        state[:] = [obs, priv, hist]
        if ev: ev[1].record()
        with torch.inference_mode():
            runner.alg.compute_returns(hist[:env.num_train_envs], priv[:env.num_train_envs])
        if ev: ev[2].record()
        out = runner.alg.update()          # returns host floats: one D2H sync per iteration
        if ev:
            ev[3].record(); torch.cuda.synchronize()
            if args.warmup <= phase_ms[3] < args.warmup + args.steps:      # the timed iterations only
                for i in range(3):
                    phase_ms[i] += ev[i].elapsed_time(ev[i + 1])
            phase_ms[3] += 1
        eb.record()
        torch.cuda.synchronize()
        spent[0] += ea.elapsed_time(eb)
        spent[1] += time.perf_counter() - tw
        return out

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    for _ in range(args.warmup):
        iteration()
    sync()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    core = env.env.core
    core.h2d_bytes = core.d2h_bytes = 0
    core.iters_counted = args.steps
    l0 = L.go1_kernel_launch_count()
    sync()
    spent[:] = [0.0, 0.0]
    prof = cprof = None
    if args.profile:
        import cProfile
        from torch.profiler import profile, ProfilerActivity
        prof = profile(activities=[ProfilerActivity.CUDA]); prof.__enter__()
        cprof = cProfile.Profile(); cprof.enable()
    for _ in range(args.steps):
        losses = iteration()
    if args.profile:
        cprof.disable(); torch.cuda.synchronize(); prof.__exit__(None, None, None)
        import pstats, io
        prof_dir = args.profile_dir or tempfile.mkdtemp(prefix="go1_bench_profile_")
        os.makedirs(prof_dir, exist_ok=True)
        with open(os.path.join(prof_dir, "kernels_torchprof.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=70))
        sio = io.StringIO(); pstats.Stats(cprof, stream=sio).sort_stats("cumulative").print_stats(45)
        with open(os.path.join(prof_dir, "host_cprofile.txt"), "w") as f:
            f.write(sio.getvalue())
        print(f"bench.py: profile written to {prof_dir}", file=sys.stderr)
    sync()
    dev_ms, wall = spent
    launches = L.go1_kernel_launch_count() - l0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, losses, state, runner)
    gemm_roof = None
    if args.gemm == 1 and not args.no_gemm_roofline:        # one more (untimed) iteration with CUDA events around every wgmma product (every rank: collectives)
        import ctypes as C
        ac_ = runner.alg.actor_critic
        streams_, ac_.update_streams = ac_.update_streams, False       # one stream: per-launch durations must not overlap to be summed
        L.go1_gemm_timing(1, None, None, None)
        iteration()
        ac_.update_streams = streams_
        ms, fl, nl = C.c_double(), C.c_double(), C.c_longlong()
        capi.check(L.go1_gemm_timing(0, C.byref(ms), C.byref(fl), C.byref(nl)), "go1_gemm_timing")
        gemm_roof = (ms.value, fl.value, nl.value)
        sync()
    t = torch.tensor([dev_ms, wall * 1e3], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, wall_ms = t.tolist()
    clocks = sampler.stop() if rank == 0 else None
    env_steps = args.steps * T_ROLLOUT * envs_per_gpu * world

    out = None
    if rank == 0:
        hbm, tf, src = peaks()
        sim_roof = sim_roofline(env, envs_per_gpu, hbm, src)
        roof = sim_roof
        if gemm_roof is not None and gemm_roof[0] > 0:
            g_ms, g_fl, g_n = gemm_roof
            ach = g_fl / (g_ms * 1e-3) / 1e12
            roof = {"bound": "tensor", "kernel": "gemm_tf32_wgmma (wgmma m64nNk8 tf32)", "achieved": ach, "peak": tf, "unit": "TFLOP/s",
                    "frac": ach / tf, "peak_source": src + ", dense TF32",
                    "scope": "every wgmma product of one PPO update + compute_returns (the rollout's products replay inside a CUDA graph)",
                    "launches": int(g_n), "kernel_ms_per_iteration": g_ms, "tflop_per_iteration": g_fl / 1e12,
                    "share_of_iteration": g_ms / (dev_ms / args.steps)}
        out = {
            "metric": METRIC, "value": env_steps / (dev_ms / 1e3), "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": dev_ms / args.steps, "higher_is_better": True, "scaling": scaling, "vs_baseline": None,
            "dtype": "f32" if args.gemm == 0 else "tf32", "data": "synthetic",
            "config": config_dict(args, world, envs_per_gpu),
            "e2e": {"value": env_steps / (wall_ms / 1e3), "unit": UNIT,
                    "h2d_bytes_per_step": int(runner_h2d_bytes(env)), "d2h_bytes_per_step": int(runner_d2h_bytes(env)) + 28,
                    "note": "on-device RL loop: actions, observations, rewards and the command curriculum never leave the GPU, so the public-API "
                            "call (Runner.rollout + compute_returns + update) copies nothing host->device and reads back only the 7 loss scalars"},
            "gpu_launches": int(launches), "clocks": clocks, "roofline": roof, "roofline_sim_step": sim_roof,
            "losses": [float(x) for x in losses[:3]],
        }
        if args.breakdown:
            n_it = args.steps
            out["phase_ms"] = {"rollout": phase_ms[0] / n_it, "compute_returns": phase_ms[1] / n_it, "update": phase_ms[2] / n_it}
        if world == 1 and not args.no_cpu_baseline:
            out["cpu_baseline"] = cpu_baseline(sample_envs=args.cpu_envs)
    del env, runner
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(out))


def runner_h2d_bytes(env):
    """Per training iteration: new commands + ids for reset/resampled envs (measured from the env's counters), env_bins."""
    c = env.env.core
    return getattr(c, "h2d_bytes", 0) / max(1, getattr(c, "iters_counted", 1))


def runner_d2h_bytes(env):
    c = env.env.core
    return getattr(c, "d2h_bytes", 0) / max(1, getattr(c, "iters_counted", 1))


def sim_roofline(env, n_envs, hbm_peak, src):
    """Fused step kernel timed alone (CUDA events on the launch stream), L2 flushed between launches."""
    import torch
    core = env.env.core
    actions = torch.zeros(n_envs, 12, device=core.device)
    flush = torch.empty(512 * 1024 * 1024 // 4, device=core.device)
    saved = [core.env_f32.clone(), core.leg_f32.clone(), core.env_i32.clone()]
    times = []
    for i in range(13):
        flush.fill_(float(i))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        core.step(actions, common_step=10_000 + i, mode=0)
        e1.record()
        torch.cuda.synchronize()
        if i >= 3:
            times.append(e0.elapsed_time(e1))
    core.env_f32.copy_(saved[0]); core.leg_f32.copy_(saved[1]); core.env_i32.copy_(saved[2])
    ms = sum(times) / len(times)
    achieved = SIM_BYTES_PER_ENV_STEP * n_envs / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": "go1_step_kernel", "achieved": achieved, "peak": hbm_peak, "unit": "GB/s", "frac": achieved / hbm_peak,
            "peak_source": src, "kernel_ms": ms, "bytes_per_env_step": SIM_BYTES_PER_ENV_STEP,
            "sim_only_env_steps_per_s": n_envs / (ms * 1e-3)}


DUMP_LIMIT_BYTES = 64 * 1024 * 1024


def dump_outputs(out_dir, losses, state, runner):
    """What the last timed iteration handed to its caller, as float32 / float64 .npy files: the loss scalars of update(), the
    observation tensors rollout() returned.  An array that would take the whole dump
    beyond 64 MB is stored as a fixed, seeded sample of its rows (the row indices are stored beside it)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"losses": np.asarray([float(x) for x in losses], dtype=np.float64)}
    for name, t in zip(("obs", "privileged_obs", "obs_history"), state):
        arrays[name] = t.detach().float().cpu().numpy()
    budget = DUMP_LIMIT_BYTES - 1024 * 1024
    per_array = budget // len(arrays)
    rng = np.random.RandomState(0)
    for name, a in arrays.items():
        if a.nbytes > per_array and a.ndim >= 1 and a.shape[0] > 1:
            rows = max(1, int(per_array // max(1, a.nbytes // a.shape[0])))
            idx = np.sort(rng.choice(a.shape[0], size=min(rows, a.shape[0]), replace=False))
            np.save(os.path.join(out_dir, name + "_rows.npy"), idx.astype(np.float64))
            a = a[idx]
        np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a))


def cpu_threads():
    """Threads of the CPU arm: the cores this process may run on, capped at 32 (torch's intra-op pool and the oracle's pthreads
    are set to the same number and never run concurrently: no oversubscription)."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    return max(1, min(n, 32))


def cpu_port_iteration(n_envs, T, threads):
    """One bounded sample of the hot path on the CPU oracle port: T-step rollout of n_envs (policy + env step) + PPO update."""
    import torch
    from env_golden_util import train_sim_config
    from oracle.env_step_oracle import OracleEnv
    from oracle.ppo_oracle import ActorCriticOracle, PPOOracle, gae
    from oracle import physics as oracle_physics
    torch.set_num_threads(threads)
    oracle_physics.set_threads(threads)
    Cfg, c, info = train_sim_config(n_envs)
    env = OracleEnv(c, info["active_reward_scales"], info["dt"], n_envs)
    ac = ActorCriticOracle()
    ppo = PPOOracle(ac)
    hist = torch.zeros(n_envs, 2100)
    t0 = time.perf_counter()
    H, P, A, V, LP, MU, R, D = [], [], [], [], [], [], [], []
    with torch.no_grad():
        priv = torch.zeros(n_envs, 2)
        for t in range(T):
            d = ac.dist(hist)
            a = d.sample()
            H.append(hist); P.append(priv); A.append(a); V.append(ac.value(hist, priv)); LP.append(d.log_prob(a).sum(-1, keepdim=True)); MU.append(d.mean)
            obs, priv, rew, reset = env.step(a)
            hist = torch.cat((hist[:, 70:], obs), -1)
            R.append(rew.unsqueeze(-1)); D.append(reset.unsqueeze(-1))
        values = torch.stack(V)
        returns, adv = gae(torch.stack(R), torch.stack(D), values, ac.value(hist, priv))
    f = lambda x: torch.stack(x).flatten(0, 1) if isinstance(x, list) else x.flatten(0, 1)
    ppo.update(f(H), f(P), f(A), f(values), f(returns), f(adv), f(LP), f(MU), torch.ones_like(f(MU)), torch.randperm(n_envs * T))
    return time.perf_counter() - t0


CPU_SAMPLE_TEXT = "{n} envs x {T}-step rollout (oracle policy + fp64 C physics + torch env logic) + full ppo_cse update on that batch"


def cpu_baseline(sample_envs=256, repeats=2):
    """The CPU port of the same path on a bounded sample: one warm-up pass, then the mean of `repeats` timed passes."""
    threads = cpu_threads()
    cpu_port_iteration(sample_envs, T_ROLLOUT, threads)
    dts = [cpu_port_iteration(sample_envs, T_ROLLOUT, threads) for _ in range(repeats)]
    dt = sum(dts) / len(dts)
    return {"value": sample_envs * T_ROLLOUT / dt, "unit": UNIT, "cores": threads, "kind": "port",
            "sample": CPU_SAMPLE_TEXT.format(n=sample_envs, T=T_ROLLOUT), "seconds_per_pass": [round(x, 2) for x in dts]}


def run_reference(args):
    """CPU port of the reference path (the reference itself needs Isaac Gym, which is not installable): rank 0 only.
    W warm-up passes, then exactly K timed passes of the same bounded sample the GPU arm's cpu_baseline uses; if the first pass
    says the whole run would not fit in ~5 minutes the sample is halved (and the line says so)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = cpu_threads()
    n_envs = args.cpu_envs
    budget_s = 300.0
    total = args.warmup + args.steps
    t_first = cpu_port_iteration(n_envs, T_ROLLOUT, threads)          # untimed (imports, thread pools)
    while n_envs > 32 and cpu_port_iteration(n_envs, T_ROLLOUT, threads) * total > budget_s:
        n_envs //= 2
    for _ in range(max(0, args.warmup - 1)):
        cpu_port_iteration(n_envs, T_ROLLOUT, threads)
    times = [cpu_port_iteration(n_envs, T_ROLLOUT, threads) for _ in range(args.steps)]
    per = sum(times) / len(times)
    v = n_envs * T_ROLLOUT / per
    world = int(os.environ.get("WORLD_SIZE", str(args.gpus)))
    scaling, envs_per_gpu = resolve_envs(args, world)
    sample = CPU_SAMPLE_TEXT.format(n=n_envs, T=T_ROLLOUT)
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": per * 1e3, "higher_is_better": True, "scaling": scaling, "vs_baseline": None, "dtype": "f32/f64",
        "data": "synthetic", "config": config_dict(args, world, envs_per_gpu),
        "sample": sample + " per timed step: a bounded sample of the config's workload on the flat-terrain CPU port",
        "cpu_baseline": {"value": v, "unit": UNIT, "cores": threads, "kind": "port",
                         "sample": sample + " (Isaac Gym is not installable: no 'reference' kind)", "first_pass_s": round(t_first, 2)},
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


def run_sweep(args, world, rank, local, device):
    """BASELINE.json configs[4]: env-count sweep (per GPU).  For every count: the fused sim-step kernel alone (L2 flushed:
    env-steps/s and algorithmic GB/s), and -- up to --sweep-train-max envs -- whole training iterations (env-steps/s)."""
    import torch
    import torch.distributed as dist
    hbm, tf, src = peaks()
    counts = [int(x) for x in args.sweep_envs.split(",")]
    rows = []
    for n in counts:
        env, runner = build_training(n, device, args.gemm, "flat")
        sim = sim_roofline(env, n, hbm, src)
        row = {"envs_per_gpu": n, "sim_kernel_ms": sim["kernel_ms"], "sim_env_steps_per_s": sim["sim_only_env_steps_per_s"] * world,
               "sim_gbs": sim["achieved"], "sim_frac_hbm": sim["frac"], "train_env_steps_per_s": None, "train_ms_per_iteration": None}
        if n <= args.sweep_train_max:
            od = env.get_observations()
            state = [od["obs"], od["privileged_obs"], od["obs_history"]]

            def iteration():
                obs, priv, hist, infos = runner.rollout(*state)
                state[:] = [obs, priv, hist]
                with torch.inference_mode():
                    runner.alg.compute_returns(hist[:env.num_train_envs], priv[:env.num_train_envs])
                return runner.alg.update()
            for _ in range(max(3, args.warmup)):
                iteration()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                iteration()
            e1.record(); torch.cuda.synchronize()
            t = torch.tensor([e0.elapsed_time(e1)], device=device, dtype=torch.float64)
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
            row["train_ms_per_iteration"] = ms / args.steps
            row["train_env_steps_per_s"] = args.steps * T_ROLLOUT * n * world / (ms / 1e3)
        rows.append(row)
        del env, runner
        torch.cuda.empty_cache()
    if world > 1:
        dist.barrier(); dist.destroy_process_group()
    if rank == 0:
        best = max((r for r in rows if r["train_env_steps_per_s"]), key=lambda r: r["train_env_steps_per_s"], default=None)
        print(json.dumps({
            "metric": METRIC, "value": best["train_env_steps_per_s"] if best else rows[-1]["sim_env_steps_per_s"], "unit": UNIT, "n_gpus": world,
            "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": best["train_ms_per_iteration"] if best else None,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32" if args.gemm == 0 else "tf32", "data": "synthetic",
            "config": {"workload": CONFIGS["sweep"]["workload"], "name": "sweep", "best_envs_per_gpu": best["envs_per_gpu"] if best else None,
                       "l2_policy": "sim step: 512 MiB L2 flush between launches; iterations: live working set > L2"},
            "sweep": rows, "roofline_peak": {"hbm_gbs": hbm, "source": src}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="flat", choices=sorted(CONFIGS), help="BASELINE.json workload (see the module docstring)")
    ap.add_argument("--scaling", default=None, choices=["weak", "strong"], help="default: the config's own (flat: weak; rough_dr, mob16k: strong)")
    ap.add_argument("--envs", type=int, default=0, help="envs per GPU (weak) or in total (strong); default: the config's own")
    ap.add_argument("--sweep-envs", default="1024,4096,16384,65536,131072", help="--config sweep: env counts per GPU")
    ap.add_argument("--sweep-train-max", type=int, default=32768, help="--config sweep: largest count that also runs whole training iterations")
    ap.add_argument("--gemm", type=int, default=int(os.environ.get("GO1_GEMM_IMPL", "1")), help="0 fp32 CUDA cores, 1 wgmma tf32")
    ap.add_argument("--cpu-envs", type=int, default=256)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gemm-roofline", action="store_true", help="skip the extra event-timed iteration (profiler runs)")
    ap.add_argument("--profile", action="store_true", help="torch.profiler (CUPTI) kernel table + cProfile of the host loop -> --profile-dir")
    ap.add_argument("--profile-dir", default=None, help="where --profile writes (default: a fresh temporary directory, named on stderr)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="after the timed steps, write what the last one returned as DIR/<name>.npy "
                    "(float32 / float64, at most 64 MB in all; larger arrays as a fixed seeded sample of rows)")
    ap.add_argument("--breakdown", action="store_true", help="per-phase CUDA-event timing (adds a sync per phase: not for headline numbers)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_b200(args)


if __name__ == "__main__":
    main()
