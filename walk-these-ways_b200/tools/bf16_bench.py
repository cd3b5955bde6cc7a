#!/usr/bin/env python
"""AC_Args.gemm_impl = 1 (TF32) against 2 (BF16 history products) on scripts/train.py's configuration, alternating the two modes after a
warm-up: ms / iteration (rollout + update, median and spread), env-steps/s, the GEMM kernel time of one update per mode
(go1_gemm_timing) and the BF16 products' achieved TFLOP/s against the H100 SXM data sheet's 989 dense; and, first, each mode's peak
memory (torch.cuda.max_memory_allocated) with only that mode's env, runner and storage alive.  Prints one JSON line with the card's name
and power limit.  --bf16-backward compares impl 2 against impl 2 with AC_Args.bf16_backward instead (keys impl2 / impl2_bf16_backward);
--csv-dir keeps each mode's per-launch GO1_GEMM_TIMING_CSV of the profiled update; --trace adds, per mode, the device time of every
kernel of one update by name (torch.profiler, a separate pass after the timed rounds) and the update's wall time.
    python walk-these-ways_b200/tools/bf16_bench.py --envs 4096 --rounds 5 [--bf16-backward] [--csv-dir DIR]"""
import argparse
import csv
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import torch  # noqa: E402


def gemm_profile(runner, L, path=None):
    """GEMM kernel time and flops of one update, split into BF16 and TF32 launches (the per-launch CSV of go1_gemm_timing)."""
    path = path or os.path.join(tempfile.mkdtemp(prefix="go1_bf16_bench_"), "gemm.csv")
    os.environ["GO1_GEMM_TIMING_CSV"] = path
    od = runner.env.get_observations()
    obs, priv, hist, _ = runner.rollout(od["obs"], od["privileged_obs"], od["obs_history"])
    L.go1_gemm_timing(1, None, None, None)
    runner.alg.compute_returns(hist, priv)
    runner.alg.update()
    ms, fl, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
    L.go1_gemm_timing(0, ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(n))
    del os.environ["GO1_GEMM_TIMING_CSV"]
    out = {"gemm_ms": ms.value, "launches": n.value, "bf16_ms": 0.0, "bf16_flop": 0.0}
    with open(path) as f:
        for r in csv.DictReader(f):
            if r.get("bf16") in ("1", "2"):
                out["bf16_ms"] += float(r["us"]) / 1e3
                out["bf16_flop"] += 2.0 * int(r["M"]) * int(r["N"]) * int(r["K"])
    out["bf16_tflops"] = out["bf16_flop"] / (out["bf16_ms"] * 1e-3) / 1e12 if out["bf16_ms"] > 0 else None
    out["bf16_frac_of_989"] = out["bf16_tflops"] / 989.0 if out["bf16_tflops"] else None
    return out


def kernel_trace(runner):
    """{kernel name: [launches, total ms]} of one update (compute_returns + update) and its wall time without the profiler."""
    from torch.profiler import ProfilerActivity, profile
    od = runner.env.get_observations()
    obs, priv, hist, _ = runner.rollout(od["obs"], od["privileged_obs"], od["obs_history"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    runner.alg.compute_returns(hist, priv)
    runner.alg.update()
    torch.cuda.synchronize()
    wall = 1e3 * (time.perf_counter() - t0)
    obs, priv, hist, _ = runner.rollout(od["obs"], od["privileged_obs"], od["obs_history"])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        runner.alg.compute_returns(hist, priv)
        runner.alg.update()
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and e.name and not e.name.startswith("Memcpy") and not e.name.startswith("Memset"):
            a = agg.setdefault(e.name[:90], [0, 0.0])
            a[0] += 1
            a[1] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    kern = dict(sorted(((k, [v[0], round(v[1], 3)]) for k, v in agg.items()), key=lambda kv: -kv[1][1]))
    return {"update_wall_ms": round(wall, 2), "update_kernel_ms": round(sum(v[1] for v in kern.values()), 2), "kernels": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3, help="iterations per timed window")
    ap.add_argument("--bf16-backward", action="store_true", help="impl 2 against impl 2 + AC_Args.bf16_backward")
    ap.add_argument("--csv-dir", default=None, help="write each mode's per-launch timing CSV here")
    ap.add_argument("--trace", action="store_true", help="per-kernel device time of one update per mode (torch.profiler)")
    a = ap.parse_args()
    modes = {"impl2": (2, False), "impl2_bf16_backward": (2, True)} if a.bf16_backward else {"impl1": (1, False), "impl2": (2, False)}

    def use(mode):
        AC_Args.gemm_impl, AC_Args.bf16_backward = modes[mode]
        return modes[mode][0]
    assert torch.cuda.is_available(), "bf16_bench needs a GPU"
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L = capi.lib()
    peak = {}
    for m in modes:              # each mode alone: build, one iteration, peak; then everything of it is freed before the other mode
        impl = use(m)
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        torch.manual_seed(0)
        env, runner = bench.build_training(a.envs, "cuda:0", impl, "flat")
        runner.learn(num_learning_iterations=1, init_at_random_ep_len=True, eval_freq=10 ** 9)
        torch.cuda.synchronize()
        peak[m] = (torch.cuda.max_memory_allocated() - base, runner.alg.storage._hist_slab.nbytes)
        del env, runner
        import gc; gc.collect()
    runners = {}
    for m in modes:
        impl = use(m)
        torch.manual_seed(0)
        env, runner = bench.build_training(a.envs, "cuda:0", impl, "flat")
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=10 ** 9)      # warm-up: graphs, packed copies, maps
        runners[m] = runner
    times = {m: [] for m in modes}
    for _ in range(a.rounds):
        for m in modes:
            use(m)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            runners[m].learn(num_learning_iterations=a.iters, eval_freq=10 ** 9)
            torch.cuda.synchronize()
            times[m].append(1e3 * (time.perf_counter() - t0) / a.iters)
    res = {"card": card, "envs": a.envs, "rounds": a.rounds, "iters_per_window": a.iters}
    for m in modes:
        use(m)
        t = times[m]
        med = statistics.median(t)
        csv_path = os.path.join(a.csv_dir, f"gemm_{m}.csv") if a.csv_dir else None
        if a.csv_dir:
            os.makedirs(a.csv_dir, exist_ok=True)
        res[m] = {"ms_per_iteration_median": round(med, 2), "ms_min": round(min(t), 2), "ms_max": round(max(t), 2),
                  "env_steps_per_s": round(a.envs * 24 / (med * 1e-3)), "peak_mem_gb": round(peak[m][0] / 2 ** 30, 3),
                  "history_slab_gb": round(peak[m][1] / 2 ** 30, 3),
                  **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in gemm_profile(runners[m], L, csv_path).items()}}
        if a.trace:
            res[m]["trace"] = kernel_trace(runners[m])
    AC_Args.gemm_impl, AC_Args.bf16_backward = 1, False
    print(json.dumps(res))


if __name__ == "__main__":
    main()
