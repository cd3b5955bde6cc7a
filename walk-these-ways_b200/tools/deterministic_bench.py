#!/usr/bin/env python
"""What AC_Args.deterministic costs: for gemm_impl 1, 2 and 2 + bf16_backward, the default and the deterministic learner on scripts/train.py's
configuration in one process, alternating after a warm-up: ms / iteration (rollout + update; median, min..max over the rounds), the GEMM
kernel time of one update (go1_gemm_timing, the deterministic products' reductions included), the device time of the added fixed-order
reduction launches (det_sum_kernel, torch.profiler in a separate pass), the growth of peak allocated memory while each runner warms up and the
deterministic workspaces the library holds.  Prints one JSON line with the card's name and power limit.
    python walk-these-ways_b200/tools/deterministic_bench.py --envs 4096 --rounds 10"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bf16_bench import bench, gemm_profile, kernel_trace  # noqa: E402
import torch  # noqa: E402

CONFIGS = {"impl1": (1, False), "impl2": (2, False), "impl2_bf16_backward": (2, True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--iters", type=int, default=3, help="iterations per timed window")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "deterministic_bench needs a GPU"
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L = capi.lib()
    runs = [(c, det) for c in CONFIGS for det in (False, True)]
    name = lambda c, det: f"{c}_{'deterministic' if det else 'default'}"

    def use(c, det):
        AC_Args.gemm_impl, AC_Args.bf16_backward = CONFIGS[c]
        AC_Args.deterministic = det
        return CONFIGS[c][0]
    runners, peak, ws = {}, {}, {}
    for c, det in runs:      # each runner built and warmed up (graphs, packed copies, maps, workspaces) while the earlier ones stay alive
        impl = use(c, det)
        torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
        base, ws0 = torch.cuda.memory_allocated(), L.go1_deterministic_workspace_bytes()
        torch.manual_seed(0)
        env, runner = bench.build_training(a.envs, "cuda:0", impl, "flat")
        assert runner.alg.actor_critic.deterministic == det
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=10 ** 9)
        torch.cuda.synchronize()
        peak[name(c, det)] = torch.cuda.max_memory_allocated() - base
        ws[name(c, det)] = L.go1_deterministic_workspace_bytes() - ws0
        runners[name(c, det)] = runner
    times = {name(c, det): [] for c, det in runs}
    for _ in range(a.rounds):
        for c, det in runs:
            use(c, det)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            runners[name(c, det)].learn(num_learning_iterations=a.iters, eval_freq=10 ** 9)
            torch.cuda.synchronize()
            times[name(c, det)].append(1e3 * (time.perf_counter() - t0) / a.iters)
    res = {"card": card, "envs": a.envs, "rounds": a.rounds, "iters_per_window": a.iters}
    for c, det in runs:
        use(c, det)
        k = name(c, det)
        t = times[k]
        g = gemm_profile(runners[k], L)
        tr = kernel_trace(runners[k])["kernels"]
        red = [v for n, v in tr.items() if "det_sum_kernel" in n]
        res[k] = {"ms_per_iteration_median": round(statistics.median(t), 2), "ms_min": round(min(t), 2), "ms_max": round(max(t), 2),
                  "update_gemm_ms": round(g["gemm_ms"], 3), "gemm_launches": g["launches"],
                  "reduction_launches": sum(v[0] for v in red), "reduction_ms": round(sum(v[1] for v in red), 3),
                  "peak_mem_growth_gb": round(peak[k] / 2 ** 30, 3), "workspace_mb": round(ws[k] / 2 ** 20, 1)}
    AC_Args.gemm_impl, AC_Args.bf16_backward, AC_Args.deterministic = 1, False, False
    print(json.dumps(res))


if __name__ == "__main__":
    main()
