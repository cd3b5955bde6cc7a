#!/usr/bin/env python
"""AC_Args.gemm_impl = 1 (TF32) against 2 (BF16 history products) on scripts/train.py's configuration, alternating the two modes after a
warm-up: ms / iteration (rollout + update, median and spread), env-steps/s, the GEMM kernel time of one update per mode
(go1_gemm_timing) and the BF16 products' achieved TFLOP/s against the H100 SXM data sheet's 989 dense; and, first, each mode's peak
memory (torch.cuda.max_memory_allocated) with only that mode's env, runner and storage alive.  Prints one JSON line with the card's name
and power limit.
    python walk-these-ways_b200/tools/bf16_bench.py --envs 4096 --rounds 5"""
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


def gemm_profile(runner, L):
    """GEMM kernel time and flops of one update, split into BF16 and TF32 launches (the per-launch CSV of go1_gemm_timing)."""
    path = os.path.join(tempfile.mkdtemp(prefix="go1_bf16_bench_"), "gemm.csv")
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
            if r.get("bf16") == "1":
                out["bf16_ms"] += float(r["us"]) / 1e3
                out["bf16_flop"] += 2.0 * int(r["M"]) * int(r["N"]) * int(r["K"])
    out["bf16_tflops"] = out["bf16_flop"] / (out["bf16_ms"] * 1e-3) / 1e12 if out["bf16_ms"] > 0 else None
    out["bf16_frac_of_989"] = out["bf16_tflops"] / 989.0 if out["bf16_tflops"] else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3, help="iterations per timed window")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bf16_bench needs a GPU"
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L = capi.lib()
    peak = {}
    for impl in (1, 2):          # each mode alone: build, one iteration, peak; then everything of it is freed before the other mode
        AC_Args.gemm_impl = impl
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        torch.manual_seed(0)
        env, runner = bench.build_training(a.envs, "cuda:0", impl, "flat")
        runner.learn(num_learning_iterations=1, init_at_random_ep_len=True, eval_freq=10 ** 9)
        torch.cuda.synchronize()
        peak[impl] = (torch.cuda.max_memory_allocated() - base, runner.alg.storage._hist_slab.nbytes)
        del env, runner
        import gc; gc.collect()
    runners = {}
    for impl in (1, 2):
        AC_Args.gemm_impl = impl
        torch.manual_seed(0)
        env, runner = bench.build_training(a.envs, "cuda:0", impl, "flat")
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=10 ** 9)      # warm-up: graphs, packed copies, maps
        runners[impl] = runner
    times = {1: [], 2: []}
    for _ in range(a.rounds):
        for impl in (1, 2):
            AC_Args.gemm_impl = impl
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            runners[impl].learn(num_learning_iterations=a.iters, eval_freq=10 ** 9)
            torch.cuda.synchronize()
            times[impl].append(1e3 * (time.perf_counter() - t0) / a.iters)
    res = {"card": card, "envs": a.envs, "rounds": a.rounds, "iters_per_window": a.iters}
    for impl in (1, 2):
        AC_Args.gemm_impl = impl
        t = times[impl]
        med = statistics.median(t)
        res[f"impl{impl}"] = {"ms_per_iteration_median": round(med, 2), "ms_min": round(min(t), 2), "ms_max": round(max(t), 2),
                              "env_steps_per_s": round(a.envs * 24 / (med * 1e-3)), "peak_mem_gb": round(peak[impl][0] / 2 ** 30, 3),
                              "history_slab_gb": round(peak[impl][1] / 2 ** 30, 3),
                              **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in gemm_profile(runners[impl], L).items()}}
    AC_Args.gemm_impl = 1
    print(json.dumps(res))


if __name__ == "__main__":
    main()
