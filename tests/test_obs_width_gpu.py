"""Observation histories of every width K0 = num_observations x num_observation_history on the tensor-core path: the pitched history roll
(go1_history_roll_pitched) bit for bit against torch.cat, HistoryWrapper's padded rows, the learner's forward and backward passes on
pitched histories against fp64 autograd, the products that must run on the tensor cores, and the training loop at observe_yaw = True
(K0 = 71 x 30 = 2130)."""
import copy
import csv
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))
SENTINEL = -7.25


@pytest.fixture(autouse=True)
def _restore_args():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    keep = AC_Args.gemm_impl
    yield
    AC_Args.gemm_impl = keep


@pytest.fixture
def gemm_csv(tmp_path, monkeypatch):
    """Runs fn between go1_gemm_timing(1) and go1_gemm_timing(0) and returns the rows of the GO1_GEMM_TIMING_CSV dump."""
    from go1_b200 import capi
    out = tmp_path / "gemm.csv"
    monkeypatch.setenv("GO1_GEMM_TIMING_CSV", str(out))

    def run(fn):
        capi.check(capi.lib().go1_gemm_timing(1, None, None, None), "timing")
        fn()
        capi.check(capi.lib().go1_gemm_timing(0, None, None, None), "timing")
        return list(csv.DictReader(open(out)))
    return run


def _roll(h, ld_in, obs, out, ld_out, n, num_obs, hist):
    from go1_b200 import capi
    return capi.lib().go1_history_roll_pitched(capi.ptr(h), ld_in, capi.ptr(obs), capi.ptr(out), ld_out, n, num_obs, hist, capi.stream_ptr())


@pytest.mark.parametrize("num_obs", [70, 71, 73, 42, 1])
def test_pitched_roll_bit_exact_vs_torch_cat(num_obs):
    """hist_out[:, :K0] == cat(hist_in[:, num_obs:K0], obs) for K0 % 4 = 0..3, with the destination's padding columns untouched (the
    source's padding holds random values that must not leak in).  Source and destination pitches differ."""
    from go1_b200 import capi
    for hist in (1, 15, 30, 31):
        K0 = num_obs * hist
        ld_in, ld_out = capi.history_pitch(K0), capi.history_pitch(K0) + 32
        for n in (1, 33, 4096):
            g = torch.Generator(device="cuda").manual_seed(n * 131 + K0)
            hbuf = torch.randn(n, ld_in, device="cuda", generator=g)
            obs = torch.randn(n, num_obs, device="cuda", generator=g)
            out = torch.full((n, ld_out), SENTINEL, device="cuda")
            capi.check(_roll(hbuf, ld_in, obs, out, ld_out, n, num_obs, hist), "roll")
            want = torch.cat((hbuf[:, num_obs:K0], obs), dim=-1)
            assert torch.equal(out[:, :K0], want), (num_obs, hist, n)
            assert bool((out[:, K0:] == SENTINEL).all()), (num_obs, hist, n)


def test_pitched_roll_rejects_bad_arguments_before_launch():
    """Short or unaligned row pitches, misaligned bases, NULL pointers and empty shapes: a non-zero return with a message, nothing written."""
    from go1_b200 import capi
    L = capi.lib()
    msg = lambda: L.go1_last_error().decode()
    n, num_obs, hist = 8, 71, 30                       # K0 = 2130, pitch 2144
    h = torch.randn(n, 2144 + 8, device="cuda")
    obs = torch.randn(n, num_obs, device="cuda")
    out = torch.full((n, 2144 + 8), SENTINEL, device="cuda")
    off = lambda t, k: C.c_void_p(t.data_ptr() + 4 * k)
    st = capi.stream_ptr()
    assert _roll(h, 2128, obs, out, 2144, n, num_obs, hist) != 0 and "ld_in 2128" in msg()
    assert _roll(h, 2144, obs, out, 2128, n, num_obs, hist) != 0 and "ld_out 2128" in msg()
    assert _roll(h, 2146, obs, out, 2144, n, num_obs, hist) != 0 and "multiples of 4" in msg()
    assert _roll(h, 2144, obs, out, 2131, n, num_obs, hist) != 0 and "multiples of 4" in msg()
    assert L.go1_history_roll_pitched(off(h, 1), 2144, capi.ptr(obs), capi.ptr(out), 2144, n, num_obs, hist, st) != 0 and "aligned" in msg()
    assert L.go1_history_roll_pitched(capi.ptr(h), 2144, capi.ptr(obs), off(out, 2), 2144, n, num_obs, hist, st) != 0 and "aligned" in msg()
    assert L.go1_history_roll_pitched(None, 2144, capi.ptr(obs), capi.ptr(out), 2144, n, num_obs, hist, st) != 0 and "null" in msg()
    assert L.go1_history_roll_pitched(capi.ptr(h), 2144, None, capi.ptr(out), 2144, n, num_obs, hist, st) != 0 and "null" in msg()
    assert L.go1_history_roll_pitched(capi.ptr(h), 2144, capi.ptr(obs), None, 2144, n, num_obs, hist, st) != 0 and "null" in msg()
    for bad in ((0, num_obs, hist), (n, 0, hist), (n, num_obs, 0), (n, -1, hist)):
        assert _roll(h, 2144, obs, out, 2144, *bad) != 0 and "positive" in msg()
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())


def _wrapper(n, num_obs, hist, seq):
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    it = iter(seq)
    env = types.SimpleNamespace(cfg=types.SimpleNamespace(env=types.SimpleNamespace(num_observation_history=hist)), num_obs=num_obs, num_envs=n,
                                device="cuda", num_privileged_obs=2)
    env.step = lambda a: (next(it), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), {"privileged_obs": torch.zeros(n, 2, device="cuda")})
    return HistoryWrapper(env)


@pytest.mark.parametrize("num_obs,hist", [(70, 15), (71, 30), (73, 31)], ids=["K1050", "K2130", "K2263"])
def test_history_wrapper_pitched_rows(num_obs, hist):
    """Four HistoryWrapper.steps equal the torch.cat chain; obs_history is a [:, :K0] view with a 16-byte row pitch and base."""
    from go1_b200 import capi
    n, K0 = 128, num_obs * hist
    seq = [torch.randn(n, num_obs, device="cuda") for _ in range(4)]
    w = _wrapper(n, num_obs, hist, seq)
    ref = torch.zeros(n, K0, device="cuda")
    for k in range(4):
        od, _, _, _ = w.step(None)
        ref = torch.cat((ref[:, num_obs:], seq[k]), dim=-1)
        h = od["obs_history"]
        assert h.shape == (n, K0) and h.stride() == (capi.history_pitch(K0), 1)
        assert h.stride(0) % 4 == 0 and h.data_ptr() % 16 == 0 and not h.is_contiguous()
        assert torch.equal(h, ref)
    for b in w._bufs:           # the padding columns stay zero
        assert bool((torch.as_strided(b, (n, b.stride(0) - K0), (b.stride(0), 1), b.storage_offset() + K0) == 0).all())


def test_history_wrapper_default_width_is_contiguous():
    """K0 = 2100 keeps contiguous 2100-float rows and the float4/float2 roll, as before."""
    n = 64
    seq = [torch.randn(n, 70, device="cuda") for _ in range(2)]
    w = _wrapper(n, 70, 30, seq)
    for k in range(2):
        od, _, _, _ = w.step(None)
        h = od["obs_history"]
        assert h.is_contiguous() and h.stride() == (2100, 1) and h.untyped_storage().nbytes() == 4 * n * 2100


# ---------------------------------------------------------------------------------------------------------------- the learner
WIDTHS = {1050: (70, 15), 2130: (71, 30), 2201: (71, 31), 2263: (73, 31)}


def _pitched_history(M, K0, seed):
    from go1_b200 import capi
    g = torch.Generator(device="cuda").manual_seed(seed)
    hbuf = torch.randn(M, capi.history_pitch(K0), device="cuda", generator=g) * 0.3
    return hbuf[:, :K0]


@pytest.mark.parametrize("M", [48, 4096])
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("E", [2, 5])
@pytest.mark.parametrize("K0", list(WIDTHS))
def test_actor_critic_matches_autograd_on_pitched_history(K0, E, impl, M):
    """forward_all + backward_ppo + backward_adaptation on a pitched history against fp64 autograd (bounds and structure of
    test_privileged_obs_gpu.test_actor_critic_matches_autograd).  M = 4096 with impl 1 runs the fused first layers."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = impl
    torch.manual_seed(K0 + E)
    NA = 12
    ac = ActorCritic(WIDTHS[K0][0], E, K0, NA).to("cuda:0")
    ac.flatten()
    h, priv = _pitched_history(M, K0, K0), torch.randn(M, E, device="cuda")
    assert ac._first_layers_fusable(h, priv) == (impl == 1 and M >= 64)
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")
    tol = 5e-3 if impl == 0 else 5e-2
    ref = {k: copy.deepcopy(getattr(ac, k)).double() for k in ("adaptation_module", "actor_body", "critic_body")}
    hd, pd = h.double(), priv.double()
    lat_ref = ref["adaptation_module"](hd)
    mean_ref, value_ref = ref["actor_body"](torch.cat((hd, lat_ref), -1)), ref["critic_body"](torch.cat((hd, pd), -1))
    close = lambda got, want: float((got.double() - want.detach()).abs().max()) < tol * (float(want.detach().abs().max()) + 1) * 2
    with torch.no_grad():
        assert close(ac.act_student(h), mean_ref)
        assert close(ac.evaluate(h, priv), value_ref)
        assert close(ac.adaptation_forward(h)[-1], lat_ref)

    ac.flat_grads.fill_(3.0)
    mean, value = ac.forward_all(h, priv, tag="train")
    assert close(mean, mean_ref) and close(value, value_ref)
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    torch.cuda.synchronize()
    grads = ac.flat_grads.clone()
    ((mean_ref * dmean.double()).sum() + (value_ref * dvalue.double()).sum()).backward()

    def check(g, mods, what):
        for nm in mods:
            for (pn, p_ref), p in zip(ref[nm].named_parameters(), getattr(ac, nm).parameters()):
                off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
                got = g[off: off + p.numel()].view_as(p)
                err = (got.double() - p_ref.grad).abs().max() / (p_ref.grad.abs().max() + 1e-12)
                assert float(err) < tol, (what, nm, pn, float(err))

    check(grads, ref, "backward_ppo")
    assert torch.equal(grads[ac.std_offset:ac.std_offset + NA], dstd)
    for mod in ref.values():
        mod.zero_grad()
    outs = ac.adaptation_forward(h)
    dpred = torch.randn(M, E, device="cuda") / M
    ac.flat_grads.fill_(3.0)
    ac.backward_adaptation(h, outs, dpred)
    torch.cuda.synchronize()
    (ref["adaptation_module"](hd) * dpred.double()).sum().backward()
    check(ac.flat_grads, ("adaptation_module",), "backward_adaptation")


def test_first_layers_run_on_tensor_cores_at_2130(gemm_csv):
    """At K0 = 2130 the update's first layers take the fused forward (one M x 1280 x 2130 product on the CTA-pair kernel) and the fused
    K-major weight gradient (1280 x (2130 + 1 + 2E) x M), as K0 = 2100 does."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 1
    torch.manual_seed(0)
    M, K0, E, NA = 4096, 2130, 2, 12
    ac = ActorCritic(71, E, K0, NA).to("cuda:0")
    ac.flatten()
    h, priv = _pitched_history(M, K0, 1), torch.randn(M, E, device="cuda")
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")

    def step():
        ac.forward_all(h, priv, tag="train")
        ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    rows = gemm_csv(step)
    shapes = {(int(r["M"]), int(r["N"]), int(r["K"])): r["kernel"] for r in rows}
    assert shapes.get((M, 1280, K0)) == "p128c2", shapes
    assert (1280, K0 + 1 + 2 * E, M) in shapes, shapes
    assert torch.isfinite(ac.flat_grads).all()


# ---------------------------------------------------------------------------------------------------------------- end to end
def _yaw_env(tmp_path, n):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from ml_logger import logger
    apply_train_config(Cfg)
    Cfg.env.observe_yaw = True
    Cfg.env.num_observations = 71
    Cfg.env.num_envs = n
    logger.configure(prefix="run", root=str(tmp_path))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    assert env.num_obs_history == 2130 and env.obs_history.stride(0) == 2144
    return env


def test_graph_replayed_rollout_equals_eager_at_observe_yaw(tmp_path, monkeypatch):
    """K0 = 2130: the graph-replayed rollout stores bit for bit what the launch-by-launch rollout stores (observations, histories,
    actions, ...), and the rollout storage keeps the padded pitch."""
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.resume)
    out = []
    try:
        for graphed in (False, True):
            torch.manual_seed(0); np.random.seed(0)
            env = _yaw_env(tmp_path, 256)
            RunnerArgs.num_steps_per_env, RunnerArgs.resume = 24, False
            runner = Runner(env, device="cuda:0")
            runner.step_graph = graphed
            if not graphed:       # launch by launch, and without the policy-only graph (its capture warm-up draws from the action-noise stream)
                runner.alg.use_cuda_graph = False
            st = runner.alg.storage
            assert st.observation_histories.shape == (24, 256, 2130) and st.observation_histories.stride(1) == 2144
            env.episode_length_buf = torch.randint(0, 1001, (256,), generator=torch.Generator().manual_seed(1))
            od = env.get_observations()
            state = (od["obs"], od["privileged_obs"], od["obs_history"])
            snaps = []
            for it in range(2):                  # the second rollout replays graphs captured during the first
                obs, priv, hist, _ = runner.rollout(*state)
                state = (obs, priv, hist)
                torch.cuda.synchronize()
                snaps.append({k: getattr(st, k).clone() for k in ("observations", "privileged_observations", "observation_histories", "actions",
                                                                  "rewards", "dones", "values", "actions_log_prob", "mu")})
                snaps[-1]["hist"] = hist.clone()
                st.clear()
            sg = runner.__dict__.get("_sg")
            assert (sg is not None and len(sg["graphs"]) == 2) if graphed else (not sg or not sg["graphs"])
            out.append(snaps)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = keep
    for it in range(2):
        assert int(out[0][it]["dones"].sum()) > 0
        assert bool((out[0][it]["observation_histories"][-1] != 0).any())
        for k in out[0][it]:
            assert torch.equal(out[0][it][k], out[1][it][k]), (it, k)


def test_policy_graph_captures_pitched_history_in_place(tmp_path, monkeypatch):
    """The rollout without the step graph replays PPO.act's policy graph; at K0 = 2130 it reads the padded history rows in place (a
    non-None history pointer in its key) instead of staging them into a contiguous copy."""
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.resume)
    try:
        env = _yaw_env(tmp_path, 256)
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = 8, False
        runner = Runner(env, device="cuda:0")
        runner.step_graph = False
        od = env.get_observations()
        runner.rollout(od["obs"], od["privileged_obs"], od["obs_history"])
        torch.cuda.synchronize()
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = keep
    keys = list(runner.alg.__dict__.get("_graph_state", {}))
    assert keys and all(k[2] is not None for k in keys), keys
    assert {k[2] for k in keys} == {b.data_ptr() for b in env._bufs}
    assert torch.isfinite(runner.alg.storage.actions).all()


def test_runner_learn_at_observe_yaw(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    env = _yaw_env(tmp_path, 256)
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = 8, 100, 1, 100, False
    try:
        runner = Runner(env, device="cuda:0")
        ac = runner.alg.actor_critic
        assert tuple(ac.actor_body[0].weight.shape) == (512, 2130 + 2)
        w0 = ac.flat_params.clone()
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=100)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = keep
    assert torch.isfinite(ac.flat_params).all() and not torch.equal(ac.flat_params, w0)
    assert np.isfinite(runner.alg._acc.cpu().numpy()).all()
