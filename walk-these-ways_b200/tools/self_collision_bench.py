#!/usr/bin/env python
"""Cost and reach of the self-collision model (Cfg.asset.model_self_collisions, DESIGN.md §3) on one GPU, in one process:

  * CUDA-event time of one fused env step (go1_step_kernel, mode 0: 4 substeps + post-physics), self-collisions off and on in
    alternating rounds, at 4096 and 65536 envs standing on flat ground under random actions, with a 512 MiB L2 flush before every
    launch (as bench.py --config sweep times the kernel);
  * ms per training iteration (24-step rollout + compute_returns + PPO update, scripts/train.py's configuration) at 4096 envs per
    mode, CUDA events around each iteration from a synchronised device, modes alternating;
  * the fraction of env-steps that end with any self-contact (a pair of the model's shapes overlapping, checked on the state after
    the step) under the shipped pretrained policy (tests/golden/pretrained_policy_fp16.*), at stance widths (commands[:, 12])
    0.10 and 0.45 m for a trot and a pace, with the model off and on;
  * the card's name and power limit.

    python walk-these-ways_b200/tools/self_collision_bench.py [--rounds 5] [--iters 5] [--warmup 2] [--out FILE.json]
"""
import argparse
import glob
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

GAITS = {"trot": (0.5, 0.0, 0.0), "pace": (0.0, 0.0, 0.5)}     # commands 5-7: phase, offset, bound (walk-these-ways' gait table)
WIDTHS = (0.10, 0.45)


def _cfg(envs, on, play=False):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    Cfg.env.num_envs = envs
    Cfg.asset.model_self_collisions = bool(on)
    if play:                   # scripts/play.py:48-61 turns the randomisation off
        dr = Cfg.domain_rand
        for k in ("push_robots", "randomize_friction", "randomize_gravity", "randomize_restitution", "randomize_motor_offset",
                  "randomize_motor_strength", "randomize_base_mass", "randomize_Kd_factor", "randomize_Kp_factor", "randomize_com_displacement"):
            setattr(dr, k, False)
    return Cfg


def step_ms(envs, on, reps=40, warmup=5):
    import torch
    from go1_b200.config import build_sim_config
    from go1_b200.sim import SimCore
    c, info = build_sim_config(_cfg(envs, on), num_envs=envs)
    assert info["self_collision"].enabled == int(on)
    sim = SimCore(c, self_collision=info["self_collision"])
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
    assert torch.isfinite(sim.leg_f32).all()
    sim.close()
    del flush
    torch.cuda.empty_cache()
    return sum(times) / len(times)


def iteration_ms(envs, on, iters, warmup):
    import numpy as np
    import torch
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    torch.manual_seed(0)
    np.random.seed(0)
    Cfg = _cfg(envs, on)
    RunnerArgs.num_steps_per_env = 24
    logger.configure(prefix="self_collision_bench", root=tempfile.mkdtemp(prefix="go1_self_collision_bench_"))
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
    del runner, env
    torch.cuda.empty_cache()
    return times


def _load_policy():
    import numpy as np
    flat, shape = {}, {}
    for fn in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "pretrained_policy_fp16.part*.npz"))):
        z = np.load(fn)
        for key in z.files:
            name, tag = key.rsplit("@", 1)
            if tag == "shape":
                shape[name] = tuple(int(v) for v in z[key])
            else:
                flat.setdefault(name, {})[int(tag)] = z[key]
    return {n: np.concatenate([c[o] for o in sorted(c)]).astype(np.float32).reshape(shape[n]) for n, c in flat.items()}


def _rot(axis, q):
    import torch
    c, s, o, z = torch.cos(q), torch.sin(q), torch.ones_like(q), torch.zeros_like(q)
    if axis == 0:
        m = [o, z, z, z, c, -s, z, s, c]
    else:
        m = [c, z, s, z, o, z, -s, z, c]
    return torch.stack(m, -1).reshape(*q.shape, 3, 3)


def _closest(p0, p1, q0, q1):
    """Batched closest points of segments (the kernel's method, DESIGN.md §3); degenerate segments are points."""
    import torch
    d1, d2, r = p1 - p0, q1 - q0, p0 - q0
    dot = lambda x, y: (x * y).sum(-1)
    a, e, f, b, c = dot(d1, d1), dot(d2, d2), dot(d2, r), dot(d1, d2), dot(d1, r)
    ap, ep = a > 0, e > 0
    sa, se = torch.where(ap, a, torch.ones_like(a)), torch.where(ep, e, torch.ones_like(e))
    den = a * e - b * b
    s = torch.where(den > 1e-6 * a * e, ((b * f - c * e) / torch.where(den > 0, den, torch.ones_like(den))).clamp(0, 1), torch.zeros_like(a))
    t = (b * s + f) / se
    s = torch.where(t < 0, (-c / sa).clamp(0, 1), torch.where(t > 1, ((b - c) / sa).clamp(0, 1), s))
    t = t.clamp(0, 1)
    s = torch.where(ap & ~ep, (-c / sa).clamp(0, 1), torch.where(~ap, torch.zeros_like(s), s))
    t = torch.where(~ap & ep, (f / se).clamp(0, 1), torch.where(~ep, torch.zeros_like(t), t))
    return p0 + s[..., None] * d1, q0 + t[..., None] * d2


def any_self_contact(core, model, sc):
    """[N] bool: some pair of the model's shapes overlaps in the current state."""
    import torch
    dev = core.device
    T = lambda x: torch.tensor(x, dtype=torch.float32, device=dev)
    pos, quat = core.env("root_pos").t(), core.env("root_quat").t()
    q = core.joint_aos("dof_pos").reshape(-1, 4, 3)
    x, y, z, w = quat.unbind(-1)
    R0 = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z),
                      2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    mv = lambda R, v: (R @ v[..., None])[..., 0]
    legs = []
    for L in range(4):
        Rw0 = R0 @ _rot(0, q[:, L, 0]); Rw1 = Rw0 @ _rot(1, q[:, L, 1]); Rw2 = Rw1 @ _rot(1, q[:, L, 2])
        p0 = pos + mv(R0, T(model["hip"][L]["origin"]).expand_as(pos))
        p1 = p0 + mv(Rw0, T(model["thigh"][L]["origin"]).expand_as(pos))
        p2 = p1 + mv(Rw1, T(model["calf"][L]["origin"]).expand_as(pos))
        pf = p2 + mv(Rw2, T(model["foot_offset"][L]).expand_as(pos))
        legs.append([(p1, p2), (p2, pf), (pf, pf)])
    rad = [sc.thigh_radius, sc.calf_radius, sc.foot_radius]
    hit = torch.zeros(pos.shape[0], dtype=torch.bool, device=dev)
    for A in range(4):
        for B in range(A + 1, 4):
            for i in range(3):
                for j in range(3):
                    c1, c2 = _closest(*legs[A][i], *legs[B][j])
                    d2 = ((c2 - c1) ** 2).sum(-1)
                    hit |= d2 < (rad[i] + rad[j]) ** 2
    h = T(model["base"]["box_half"])
    for L in range(4):
        (p1, p2), (_, pf), _ = legs[L]
        for k, c in enumerate((p2, 0.5 * (p2 + pf), pf)):
            lc = (R0.transpose(1, 2) @ (c - pos)[..., None])[..., 0]
            d = lc - torch.maximum(torch.minimum(lc, h), -h)
            hit |= (d * d).sum(-1) < rad[k] ** 2
    return hit


def contact_rate(on, gait, width, n=256, steps=250, skip=20):
    import torch
    from go1_b200.config import load_model, self_collision_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import ActorCritic
    Cfg = _cfg(n, on, play=True)
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    sc = self_collision_config(Cfg)
    model = load_model()
    ac = ActorCritic(env.num_obs, env.num_privileged_obs, env.num_obs_history, env.num_actions).to("cuda:0")
    sd = ac.state_dict()
    for k, v in _load_policy().items():
        sd[k] = torch.from_numpy(v)
    ac.load_state_dict(sd)
    obs = env.reset()
    hits, total, resets = 0, 0, 0
    ph, off, bd = GAITS[gait]
    for i in range(steps):
        with torch.no_grad():
            actions = ac.act_student(obs["obs_history"]).clone()
        c = env.commands
        c[:, 0] = 1.0; c[:, 1] = 0.0; c[:, 2] = 0.0; c[:, 3] = 0.0; c[:, 4] = 3.0
        c[:, 5] = ph; c[:, 6] = off; c[:, 7] = bd; c[:, 8] = 0.5; c[:, 9] = 0.08; c[:, 10] = 0.0; c[:, 11] = 0.0; c[:, 12] = width
        obs, rew, done, info = env.step(actions)
        if i >= skip:
            hits += int(any_self_contact(env.env.core, model, sc).sum())
            total += n
            resets += int(done.sum())
    del ac, env
    torch.cuda.empty_cache()
    return {"contact_fraction": round(hits / total, 4), "resets": resets, "env_steps": total}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iter-rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "self_collision_bench measures on cuda:0 (no CPU fallback)"
    res = {"card": card(), "rounds": args.rounds, "step_kernel_ms": {}, "iteration_ms": {}, "contact_fraction": {}}
    for envs in (4096, 65536):
        t = {"off": [], "on": []}
        for r in range(args.rounds):
            for mode in ("off", "on"):
                t[mode].append(step_ms(envs, mode == "on"))
        res["step_kernel_ms"][envs] = {m: {"median": round(sorted(v)[len(v) // 2], 4), "min": round(min(v), 4), "max": round(max(v), 4)}
                                       for m, v in t.items()}
        print(f"{envs} envs step kernel: {res['step_kernel_ms'][envs]}", file=sys.stderr, flush=True)
    it = {"off": [], "on": []}
    for r in range(args.iter_rounds):
        for mode in ("off", "on"):
            it[mode] += iteration_ms(4096, mode == "on", args.iters, args.warmup)
    res["iteration_ms"] = {m: {"median": round(sorted(v)[len(v) // 2], 2), "min": round(min(v), 2), "max": round(max(v), 2), "n": len(v)}
                           for m, v in it.items()}
    print(f"iteration: {res['iteration_ms']}", file=sys.stderr, flush=True)
    for gait in GAITS:
        for w in WIDTHS:
            for mode in ("off", "on"):
                res["contact_fraction"][f"{gait}/{w}/{mode}"] = contact_rate(mode == "on", gait, w)
                print(f"{gait} {w} {mode}: {res['contact_fraction'][f'{gait}/{w}/{mode}']}", file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
