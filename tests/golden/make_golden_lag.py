#!/usr/bin/env python
"""Generates tests/golden/lag.npz by running the REFERENCE's own LeggedRobot._compute_torques (imported through tests/_stubs, on
make_golden.mock_env with scripts/train.py's config) for every Cfg.domain_rand.lag_timesteps case of lag_util.CASES:

    python tests/golden/make_golden_lag.py

Per case `c` the env starts from lag_util.inputs(c) (re-created by the tests, not stored) with lag_buffer = [zeros] + the L seeded
slots, and runs lag_util.T policy steps of `decimation` substeps each.  Per substep k (= step * decimation + substep) the file holds
"c/target" [k][N][12] (joint_pos_target), "c/torque" [k][N][12] and "c/fifo" [k][L][N][12] (the L live slots after the substep).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))      # lag_util
import make_golden  # noqa: E402  (puts the stubs and the reference on sys.path)
import torch  # noqa: E402

import lag_util as U  # noqa: E402


def run(Cfg, case, out):
    from go1_gym.envs.base.legged_robot import LeggedRobot
    L, control_type, decimation = U.CASES[case]
    Cfg.domain_rand.randomize_lag_timesteps = True
    Cfg.domain_rand.lag_timesteps = L
    Cfg.control.control_type = control_type
    Cfg.control.decimation = 4                 # mock_env derives dt from 4 substeps; only the substep count below changes
    env = make_golden.mock_env(Cfg, U.N, torch.Generator().manual_seed(0))
    x = {k: torch.from_numpy(v) for k, v in U.inputs(case, env.default_dof_pos[0].numpy()).items()}
    for k in ("dof_pos", "dof_vel", "joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last", "joint_vel_last_last", "motor_offsets"):
        setattr(env, k, x[k].clone())
    env.motor_strengths = x["motor_strengths"][:, None].repeat(1, 12)
    env.lag_buffer = [torch.zeros(U.N, 12)] + [x["fifo"][i].clone() for i in range(L)]
    tgt, tq, fifo = [], [], []
    with torch.no_grad():
        for t in range(U.T):
            for _ in range(decimation):
                tq.append(LeggedRobot._compute_torques(env, x["actions"][t].clone()).view(U.N, 12).numpy().copy())
                tgt.append(env.joint_pos_target.numpy().copy())
                fifo.append(torch.stack(env.lag_buffer[1:]).numpy().copy() if L else np.zeros((0, U.N, 12), np.float32))
    assert len(env.lag_buffer) == L + 1
    out[f"{case}/target"], out[f"{case}/torque"], out[f"{case}/fifo"] = np.stack(tgt), np.stack(tq), np.stack(fifo)
    print(case, "torque range", float(np.abs(out[f"{case}/torque"]).max()))


def main():
    Cfg, _ = make_golden.reference_train_cfg()
    out = {}
    for case in U.CASES:
        run(Cfg, case, out)
    path = os.path.join(HERE, "lag.npz")
    np.savez_compressed(path, **out)
    print("lag.npz:", len(out), "arrays,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
