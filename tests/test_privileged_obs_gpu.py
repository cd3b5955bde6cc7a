"""num_privileged_obs up to 64 on the learner kernels: the trailing-input kernels (go1_mlp_extra_forward / go1_mlp_extra_backward) against
fp64, ActorCritic's forward and backward passes against fp64 autograd on both routes (layer by layer and the fused first layers), a full
PPO cycle against the reference's own vectors (tests/golden/ppo_priv.npz), and Runner.learn with every privileged group."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))
import priv_obs_util as U  # noqa: E402
from activation_test_util import KINDS, MODULES  # noqa: E402

pytestmark = pytest.mark.gpu
ES = [1, 4, 5, 8, 13, 18, 45, 64]

# every privileged-observation group of the reference's compute_observations (45 columns), and friction + restitution + body velocity
ALL_GROUPS = ("friction", "restitution", "base_mass", "com_displacement", "motor_strength", "motor_offset", "body_height", "body_velocity",
              "gravity", "clock_inputs", "desired_contact_states")
ESTIMATION_GROUPS = ("friction", "restitution", "body_velocity")


@pytest.fixture(autouse=True)
def _restore_args():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    from go1_gym_learn.ppo_cse.ppo import PPO_Args
    keep = {k: copy.copy(getattr(AC_Args, k)) for k in ("activation", "gemm_impl", "actor_hidden_dims", "critic_hidden_dims", "adaptation_module_branch_hidden_dims")}
    sel = PPO_Args.selective_adaptation_module_loss
    yield
    for k, v in keep.items():
        setattr(AC_Args, k, v)
    PPO_Args.selective_adaptation_module_loss = sel


def _lib():
    from go1_b200 import capi
    return capi, capi.lib(), capi.stream_ptr()


def _strided(rows, cols, lead, scale=1.0, seed=0):
    """A [rows][cols] view at column `lead` of a wider buffer: row stride lead + cols + 1 (not a multiple of 4 floats for most cols)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(rows, lead + cols + 1, device="cuda", generator=g) * scale
    return buf[:, lead:lead + cols]


@pytest.mark.parametrize("M", [1, 63, 4097])
@pytest.mark.parametrize("E", ES)
def test_extra_forward_matches_fp64(E, M):
    """y = f(y + extra W_e^T) in place for every activation kind (and none), float4 rows and scalar rows (o % 4 != 0 or a misaligned
    row stride), strided extra and W_e (W_e a slice of a wider first-layer weight, as in ActorCritic)."""
    capi, L, st = _lib()
    ex = _strided(M, E, 3, seed=E)
    for o, pad in ((512, 0), (256, 4), (100, 1), (37, 0)):
        W = _strided(o, E, 2100, scale=0.3, seed=o)
        y0 = torch.randn(M, o + pad, device="cuda")[:, :o]
        pre = y0.double() + ex.double() @ W.double().t()
        mag = y0.double().abs() + ex.double().abs() @ W.double().abs().t()
        for kind in [None] + list(KINDS):
            y = y0.clone() if pad == 0 else torch.randn(M, o + pad, device="cuda")[:, :o].copy_(y0)
            act = 0 if kind is None else capi.act_arg(capi.ACTIVATIONS[kind], 1)
            capi.check(L.go1_mlp_extra_forward(capi.ptr(y), y.stride(0), capi.ptr(ex), ex.stride(0), capi.ptr(W), W.stride(0), M, o, E, act, st), "extra_fwd")
            ref = pre if kind is None else MODULES[kind]()(pre)
            bound = 2e-6 + 2e-6 * mag * 1.06      # fp32 sums of E + 1 terms, and act_fast's 1e-6 (selu stretches by 1.05)
            err = (y.double() - ref).abs()
            assert bool((err <= bound).all()), (o, pad, kind, float(err.max()))


@pytest.mark.parametrize("M", [1, 63, 4097])
@pytest.mark.parametrize("E", ES)
def test_extra_backward_matches_fp64(E, M):
    """d(extra) = dz W_e from a row-major dz [M][o] and from a transposed one [o][M] (the first-layer dz of the fused backward), and the
    weight gradient g_W_e = dz^T extra (overwriting: the output is filled with 3.0 first), with strided operands."""
    capi, L, st = _lib()
    ex = _strided(M, E, 3, seed=E + 1)
    for o in (512, 130):
        W = _strided(o, E, 2100, scale=0.3, seed=o + 1)
        dz = torch.randn(M, o, device="cuda") / 8
        dzT = torch.zeros(o, (M + 31) // 32 * 32 + 4, device="cuda")
        dzT[:, :M] = dz.t()
        want_dx = dz.double() @ W.double()
        bound_dx = 1e-5 * (dz.double().abs() @ W.double().abs()) + 1e-6
        want_gw = dz.double().t() @ ex.double()
        bound_gw = 1e-5 * (dz.double().abs().t() @ ex.double().abs()) + 1e-6
        gbuf = torch.full((o, 9 + E + 2), 3.0, device="cuda")
        gw = gbuf[:, 9:9 + E]
        for transposed, d, ldd in ((0, dz, dz.stride(0)), (1, dzT, dzT.stride(0))):
            dx = torch.full((M, E + 2), 3.0, device="cuda")[:, :E]
            g_ptr = capi.ptr(gw) if not transposed else None
            capi.check(L.go1_mlp_extra_backward(capi.ptr(d), ldd, transposed, capi.ptr(ex), ex.stride(0), capi.ptr(W), W.stride(0), g_ptr, gw.stride(0),
                                                capi.ptr(dx), dx.stride(0), M, o, E, 0, st), "extra_backward")
            err = (dx.double() - want_dx).abs()
            assert bool((err <= bound_dx).all()), (o, transposed, float(err.max()))
        err = (gw.double() - want_gw).abs()
        assert bool((err <= bound_gw).all()), (o, float(err.max()))
        assert bool((gbuf[:, :9] == 3.0).all() and (gbuf[:, 9 + E:] == 3.0).all())
        # accumulate = 1 adds into the output; the weight gradient alone (dextra NULL)
        capi.check(L.go1_mlp_extra_backward(capi.ptr(dz), dz.stride(0), 0, capi.ptr(ex), ex.stride(0), None, 0, capi.ptr(gw), gw.stride(0), None, 0,
                                            M, o, E, 1, st), "extra_backward")
        err = (gw.double() - 2 * want_gw).abs()
        assert bool((err <= 2 * bound_gw).all()), (o, "accumulate", float(err.max()))


def test_bad_arguments_are_rejected_before_launch():
    """E = 65, NULL pointers, short row strides and a weight gradient from a transposed dz: non-zero return code and a message, and
    nothing written."""
    capi, L, st = _lib()
    msg = lambda: L.go1_last_error().decode()
    x = torch.zeros(128, 128, device="cuda")
    p = capi.ptr(x)
    assert L.go1_mlp_extra_forward(p, 128, p, 65, p, 65, 64, 64, 65, 1, st) != 0 and "1..64" in msg()
    assert L.go1_mlp_extra_forward(None, 128, p, 8, p, 8, 64, 64, 8, 1, st) != 0
    assert L.go1_mlp_extra_forward(p, 128, p, 4, p, 8, 64, 64, 8, 1, st) != 0 and "stride" in msg()
    assert L.go1_mlp_extra_forward(p, 32, p, 8, p, 8, 64, 64, 8, 1, st) != 0 and "stride" in msg()
    assert L.go1_mlp_extra_backward(p, 128, 0, p, 65, p, 65, p, 65, p, 65, 64, 64, 65, 0, st) != 0 and "1..64" in msg()
    assert L.go1_mlp_extra_backward(None, 128, 0, p, 8, p, 8, p, 8, p, 8, 64, 64, 8, 0, st) != 0
    assert L.go1_mlp_extra_backward(p, 128, 0, p, 8, p, 8, None, 8, None, 8, 64, 64, 8, 0, st) != 0 and "nothing" in msg()
    assert L.go1_mlp_extra_backward(p, 128, 0, p, 8, None, 8, None, 8, p, 8, 64, 64, 8, 0, st) != 0 and "w_extra" in msg()
    assert L.go1_mlp_extra_backward(p, 128, 0, p, 4, p, 8, p, 8, None, 8, 64, 64, 8, 0, st) != 0 and "ldex" in msg()
    assert L.go1_mlp_extra_backward(p, 128, 1, p, 8, p, 8, p, 8, None, 8, 64, 64, 8, 0, st) != 0 and "dz_transposed" in msg()
    assert L.go1_mlp_extra_backward(p, 32, 1, p, 8, p, 8, None, 8, p, 8, 64, 64, 8, 0, st) != 0 and "lddz" in msg()
    torch.cuda.synchronize()
    assert bool((x == 0).all())


def _ref_modules(ac):
    return {k: copy.deepcopy(getattr(ac, k)).double() for k in ("adaptation_module", "actor_body", "critic_body")}


@pytest.mark.parametrize("M", [48, 4096])
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("E", [5, 18, 45])
def test_actor_critic_matches_autograd(E, impl, M):
    """forward_all + backward_ppo + backward_adaptation at the default layer shapes against fp64 autograd.  M = 48: layer by layer;
    M = 4096 with impl 1: the fused first layers (one packed forward product, the transposed first-layer dz and the K-major weight gradient
    with 2E augmented rows).  The gradient buffer is filled with 3.0 first: both backward passes overwrite their region.  Every other
    forward entry point is checked against the same modules."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = impl
    torch.manual_seed(3)
    NOBS, NH, NA = 70, 2100, 12
    ac = ActorCritic(NOBS, E, NH, NA).to("cuda:0")
    ac.flatten()
    hbuf = torch.randn(M, 2112, device="cuda") * 0.3      # the minibatch pitch RolloutStorage uses
    h, priv = hbuf[:, :NH], torch.randn(M, E, device="cuda")
    assert ac._first_layers_fusable(h, priv) == (impl == 1 and M >= 64)
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")
    tol = 5e-3 if impl == 0 else 5e-2

    ref = _ref_modules(ac)
    hd, pd = h.double(), priv.double()
    lat_ref = ref["adaptation_module"](hd)
    mean_ref, value_ref = ref["actor_body"](torch.cat((hd, lat_ref), -1)), ref["critic_body"](torch.cat((hd, pd), -1))
    close = lambda got, want: float((got.double() - want.detach()).abs().max()) < tol * (float(want.detach().abs().max()) + 1) * 2
    with torch.no_grad():
        assert close(ac.act_student(h), mean_ref)
        assert close(ac.act_teacher(h, priv), ref["actor_body"](torch.cat((hd, pd), -1)))
        assert close(ac.evaluate(h, priv), value_ref)
        assert close(ac.get_student_latent(h), lat_ref)
        assert close(ac.adaptation_forward(h)[-1], lat_ref)
        a = ac.act(h)
        assert a.shape == (M, NA) and torch.isfinite(a).all() and close(ac.action_mean, mean_ref)

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
    assert bool((grads[ac.HEAD:] != 3.0).any())
    for mod in ref.values():
        mod.zero_grad()
    outs = ac.adaptation_forward(h)
    dpred = torch.randn(M, E, device="cuda") / M
    ac.flat_grads.fill_(3.0)
    ac.backward_adaptation(h, outs, dpred)
    torch.cuda.synchronize()
    (ref["adaptation_module"](hd) * dpred.double()).sum().backward()
    check(ac.flat_grads, ("adaptation_module",), "backward_adaptation")


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("case", list(U.CASES))
def test_full_ppo_cycle_matches_reference_vectors(case, impl):
    """act x24 -> process_env_step -> compute_returns -> update on the reference's own vectors (default network, minibatches of 96 rows:
    the fused first layers with impl 1) for 5, 18 and 45 privileged observations and the selective adaptation loss.  Tolerances as in
    test_activations_gpu.test_full_ppo_cycle_matches_reference_vectors."""
    from ppo_golden_util import seeded_weights, sample_tensor
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO, PPO_Args
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    g = np.load(os.path.join(HERE, "golden", "ppo_priv.npz"))
    inp = U.inputs()
    E, selective = U.CASES[case]
    AC_Args.gemm_impl = impl
    PPO_Args.selective_adaptation_module_loss = selective
    k = 1.0 if impl == 0 else 250.0
    ac = ActorCritic(U.NOBS, E, U.NH, U.NA)
    w = seeded_weights({kk: tuple(v.shape) for kk, v in ac.state_dict().items()})
    ac.load_state_dict({kk: torch.from_numpy(v) for kk, v in w.items()})
    alg = PPO(ac, device="cuda:0")
    alg.init_storage(U.N, U.T, [U.NOBS], [E], [U.NH], [U.NA])
    C = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for t in range(U.T):
        ac.injected_eps = C(inp["in/eps"][t])
        alg.act(C(inp["in/obs"][t]), C(inp["in/priv"][t][:, :E]), C(inp["in/hist"][t]))
        infos = {"env_bins": torch.zeros(U.N, device="cuda"), "time_outs": torch.zeros(U.N, dtype=torch.bool, device="cuda")}
        alg.process_env_step(C(inp["in/rew"][t]), C(inp["in/done"][t]), infos)
    alg.compute_returns(C(inp["last/hist"]), C(inp["last/priv"][:, :E]))
    st = alg.storage
    for nm, tol in (("actions", 2e-5), ("values", 2e-5), ("actions_log_prob", 1e-4), ("mu", 2e-5), ("returns", 5e-5), ("advantages", 2e-4)):
        got, want = getattr(st, nm).cpu().numpy(), g[f"{case}/storage/{nm}"]
        assert np.allclose(got, want, rtol=1e-4 * k, atol=tol * k), (nm, np.abs(got - want).max())
    alg.fixed_minibatch_indices = C(inp["in/perm"])
    losses = alg.update()
    ref = g[f"{case}/update/losses"]
    kl = 1.0 if impl == 0 else 25.0
    assert abs(losses[0] - ref[0]) < 2e-3 * kl * abs(ref[0]) and abs(losses[1] - ref[1]) < 2e-3 * kl and abs(losses[2] - ref[2]) < 2e-3 * kl * abs(ref[2])
    assert abs(losses[5] - ref[5]) < 2e-3 * kl * abs(ref[5])
    if impl == 0:
        assert abs(alg.learning_rate - float(g[f"{case}/update/learning_rate"])) < 1e-12
    for name_k, v in ac.state_dict().items():
        got, want = sample_tensor(v.cpu().numpy(), stride=U.sample_stride(v.numel())), g[f"{case}/final/{name_k}"]
        if impl == 0:
            assert np.allclose(got[:-2], want[:-2], rtol=0, atol=3e-4), (name_k, np.abs(got[:-2] - want[:-2]).max())
        else:
            d = np.abs(got[:-2] - want[:-2])
            assert np.quantile(d, 0.99) < 4e-3 and d.max() < 4e-2, (name_k, np.quantile(d, 0.99), d.max())


def test_graph_replayed_act_matches_eager_with_45_privileged_obs():
    """PPO.act's captured CUDA graph (the rollout path) gives the eager pass's actions and values with E = 45."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 1
    torch.manual_seed(4)
    M, E = 4096, 45
    ac = ActorCritic(70, E, 2100, 12)
    alg = PPO(ac, device="cuda:0")
    h, priv = torch.randn(M, 2100, device="cuda") * 0.3, torch.randn(M, E, device="cuda")
    ac.injected_eps = torch.randn(M, 12, device="cuda")
    a_eager, v_eager = (t.clone() for t in alg._act_eager(h, priv))
    for _ in range(2):          # capture, then replay
        a_graph, v_graph = alg._act_graphed(h, priv)
    torch.cuda.synchronize()
    assert torch.allclose(a_graph, a_eager, rtol=0, atol=1e-6) and torch.allclose(v_graph, v_eager, rtol=0, atol=1e-6)


@pytest.mark.parametrize("groups", [ALL_GROUPS, ESTIMATION_GROUPS], ids=["all45", "estimation5"])
def test_runner_learn_with_privileged_groups(groups, tmp_path, monkeypatch):
    """scripts/train.py's flow with the given priv_observe_* groups: a short Runner.learn (graph-replayed rollout) trains, and the
    TorchScript artefacts scripts/play.py loads reproduce the inference policy."""
    monkeypatch.chdir(tmp_path)
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    from ml_logger import logger
    apply_train_config(Cfg)
    widths = {"friction": 1, "restitution": 1, "base_mass": 1, "com_displacement": 3, "motor_strength": 12, "motor_offset": 12, "body_height": 1,
              "body_velocity": 3, "gravity": 3, "clock_inputs": 4, "desired_contact_states": 4}
    for name in groups:
        setattr(Cfg.env, "priv_observe_" + name, True)
    Cfg.env.num_privileged_obs = sum(widths[n] for n in groups)
    Cfg.env.num_envs = 256
    logger.configure(prefix="run", root=str(tmp_path))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    assert env.num_privileged_obs == Cfg.env.num_privileged_obs
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = 8, 1, 1, 100, False
    try:
        runner = Runner(env, device="cuda:0")
        ac = runner.alg.actor_critic
        assert ac.num_privileged_obs == Cfg.env.num_privileged_obs
        w0 = ac.flat_params.clone()
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=100)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = keep
    assert torch.isfinite(ac.flat_params).all() and not torch.equal(ac.flat_params, w0)
    assert np.isfinite(runner.alg._acc.cpu().numpy()).all()
    ck = os.path.join(str(tmp_path), "run", "checkpoints")
    body = torch.jit.load(os.path.join(ck, "body_latest.jit"))
    adapt = torch.jit.load(os.path.join(ck, "adaptation_module_latest.jit"))
    h = torch.randn(5, env.num_obs_history) * 0.3
    policy = runner.get_inference_policy(device="cuda:0")
    AC_Args.gemm_impl = 0      # the exact-fp32 kernels against TorchScript's fp32 on the CPU
    want = policy({"obs_history": h.cuda()}).cpu()
    got = body(torch.cat((h, adapt(h)), dim=-1))
    assert torch.allclose(got, want, rtol=1e-4, atol=2e-5), float((got - want).abs().max())
