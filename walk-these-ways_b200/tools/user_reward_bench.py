#!/usr/bin/env python
"""Cost of user reward terms (go1_gym/envs/rewards, DESIGN.md §4) on one GPU, in one process:

  * ms per env step (LeggedRobot.step with the device curriculum: step launch(es), resample, reset, fold), CUDA events around a
    window of steps, for K = 0, 1 and 4 cheap user terms at 4096 and 65536 envs under random actions, arms alternating by round;
  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration) for the same arms,
    CUDA events around each iteration from a synchronised device, arms alternating by round.  At 65536 envs three runners'
    rollout storage does not fit on one 80 GB card, so each round builds, warms up, times and frees one runner per arm in turn;
  * every round's time next to the medians, so the round-to-round spread can be compared with the differences between arms;
  * the card's name and power limit.

K = 0 is the plain kernel; K = 1 adds one term computed in torch; K = 4 adds four.

    python walk-these-ways_b200/tools/user_reward_bench.py [--envs 4096 65536] [--rounds 5] [--steps 100] [--iters 3] [--out FILE.json]
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

ARMS = (0, 1, 4)


def _container(K):
    import torch
    from go1_gym.envs.rewards import REWARD_CONTAINERS, CoRLRewards

    class Bench(CoRLRewards):
        def _reward_u0(self):
            return torch.square(self.env.base_lin_vel[:, 2])

        def _reward_u1(self):
            return torch.sum(torch.square(self.env.base_ang_vel[:, :2]), dim=1)

        def _reward_u2(self):
            return torch.sum(torch.square(self.env.last_actions - self.env.actions), dim=1)

        def _reward_u3(self):
            return torch.sum(torch.square(self.env.dof_vel), dim=1)

    name = f"UserRewardBench{K}"
    REWARD_CONTAINERS[name] = type(name, (Bench,), {})
    return name


def _env(envs, K):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    apply_train_config(Cfg)
    Cfg.env.num_envs = envs
    Cfg.rewards.reward_container_name = _container(K)
    for k in range(K):
        setattr(Cfg.reward_scales, f"u{k}", -0.01)
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    assert len(env.env.user_reward_names) == K
    return env


def step_ms(envs, rounds, steps):
    import torch
    arms = {K: _env(envs, K) for K in ARMS}
    gen = torch.Generator(device="cuda").manual_seed(0)
    a = torch.empty(envs, 12, device="cuda")
    for env in arms.values():
        env.reset()
        for _ in range(10):
            env.step(a.normal_(generator=gen))
    times = {K: [] for K in ARMS}
    for _ in range(rounds):
        for K, env in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                env.step(a.normal_(generator=gen))
            e1.record()
            torch.cuda.synchronize()
            times[K].append(e0.elapsed_time(e1) / steps)
    del arms, env
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    return {K: sorted(v)[len(v) // 2] for K, v in times.items()}, times


def iteration_ms(envs, rounds, warmup, alternate):
    """alternate: all three runners live at once and take turns; otherwise (rollout storage of three runners at 65536 envs does not
    fit in 80 GB) every round builds and warms up a fresh runner per arm, arms in turn."""
    import gc
    import torch
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    logger.configure(prefix="user_reward_bench", root=tempfile.mkdtemp())
    RunnerArgs.resume, RunnerArgs.save_video_interval, RunnerArgs.save_interval, RunnerArgs.log_freq = False, 10 ** 9, 10 ** 9, 10 ** 9

    def make(K):
        r = Runner(_env(envs, K), device="cuda:0")
        r.save = lambda it: None
        r.learn(num_learning_iterations=warmup, init_at_random_ep_len=True)
        return r

    def one(r):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r.learn(num_learning_iterations=1)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    times, graphed = {K: [] for K in ARMS}, {}
    if alternate:
        runners = {K: make(K) for K in ARMS}
        for _ in range(rounds):
            for K, r in runners.items():
                times[K].append(one(r))
        graphed = {K: r._sg is not None for K, r in runners.items()}
        del runners
    else:
        for _ in range(rounds):
            for K in ARMS:
                r = make(K)
                times[K].append(one(r))
                graphed[K] = r._sg is not None
                del r
                gc.collect()
                torch.cuda.empty_cache()
    gc.collect()
    torch.cuda.empty_cache()
    return {K: sorted(v)[len(v) // 2] for K, v in times.items()}, times, graphed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("user_reward_bench.py needs a CUDA device")
    out = os.path.abspath(args.out) if args.out else None
    os.chdir(tempfile.mkdtemp())            # Runner.save / the logger write relative paths
    res = {"card": card(), "step_ms": {}, "step_ms_rounds": {}, "iteration_ms": {}, "iteration_ms_rounds": {}, "iteration_graphed": {}}
    for envs in args.envs:
        res["step_ms"][envs], res["step_ms_rounds"][envs] = step_ms(envs, args.rounds, args.steps)
        print(f"{envs} envs, env step ms by K: {res['step_ms'][envs]} rounds {res['step_ms_rounds'][envs]}", file=sys.stderr, flush=True)
        res["iteration_ms"][envs], res["iteration_ms_rounds"][envs], res["iteration_graphed"][envs] = \
            iteration_ms(envs, args.iters, args.warmup, alternate=envs <= 16384)
        print(f"{envs} envs, iteration ms by K: {res['iteration_ms'][envs]} rounds {res['iteration_ms_rounds'][envs]} "
              f"(graphed: {res['iteration_graphed'][envs]})", file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
