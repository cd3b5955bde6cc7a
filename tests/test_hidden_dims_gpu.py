"""AC_Args hidden-layer shapes (actor_hidden_dims, critic_hidden_dims, adaptation_module_branch_hidden_dims) on the tensor-core path:
the learner's forward and backward passes against fp64 autograd, every ragged fused-tail instantiation against fp64 through the C ABI,
the products of an update (all on the tensor cores, the tails fused), the graph-replayed PPO.act and a full PPO cycle against the
reference's vectors (tests/golden/ppo_hidden.npz)."""
import copy
import csv
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))

# (actor = critic hidden dims, adaptation module hidden dims)
SHAPES = {
    "default": ([512, 256, 128], [256, 128]),
    "wide": ([1024, 512, 256], [512, 256]),
    "narrow": ([256, 128, 64], [128, 64]),
    "deep": ([512, 256, 128, 64], [256, 128]),
    "ragged": ([500, 250, 125], [250, 125]),
    "one_layer": ([256], [64]),
    "w36_250": ([250, 36], [36, 250]),
    "small_last": ([64, 50, 36, 20], [40, 25]),       # last hidden widths below 32: the heads' wgrads on the skinny kernel
    "tiny": ([256, 4, 64], [128, 6]),                  # inputs narrower than 8 floats into a tensor-core wgrad
}
NOBS, K0, NA = 70, 280, 12


@pytest.fixture(autouse=True)
def _restore_ac_args():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    keep = {k: copy.copy(getattr(AC_Args, k)) for k in ("activation", "gemm_impl", "actor_hidden_dims", "critic_hidden_dims", "adaptation_module_branch_hidden_dims")}
    yield
    for k, v in keep.items():
        setattr(AC_Args, k, v)


def _make(shape, E, impl, activation="elu", critic=None, seed=0):
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    hidden, adapt = SHAPES[shape]
    AC_Args.gemm_impl, AC_Args.activation = impl, activation
    AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims = list(hidden), list(critic or hidden), list(adapt)
    torch.manual_seed(seed)
    ac = ActorCritic(NOBS, E, K0, NA).to("cuda:0")
    ac.flatten()
    return ac


def _check_against_autograd(ac, M, E, impl, activation):
    h, priv = torch.randn(M, K0, device="cuda") * 0.3, torch.randn(M, E, device="cuda")
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


@pytest.mark.parametrize("M", [48, 4096])
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("act_E", [("elu", 2), ("elu", 5), ("tanh", 2), ("sigmoid", 5)], ids=lambda v: f"{v[0]}-E{v[1]}")
@pytest.mark.parametrize("shape", list(SHAPES))
def test_actor_critic_matches_autograd(shape, act_E, impl, M):
    """forward_all, backward_ppo and backward_adaptation against fp64 autograd (bounds of test_obs_width_gpu); M = 4096 with impl 1 runs
    the fused first layers and the fused tails."""
    activation, E = act_E
    ac = _make(shape, E, impl, activation, seed=M + E)
    _check_against_autograd(ac, M, E, impl, activation)


@pytest.mark.parametrize("impl", [0, 1])
def test_actor_critic_matches_autograd_at_minibatch_rows(impl):
    """The update's minibatch size at 4096 environments (M = 24576) on a ragged shape."""
    ac = _make("ragged", 2, impl)
    _check_against_autograd(ac, 24576, 2, impl, "elu")


def test_wide_latent_head_matches_autograd():
    """An adaptation head wider than the skinny kernels take (E = 18), behind a 6-wide hidden layer: its gradient rows are copied to a
    padded buffer for the tensor-core wgrad and dgrad."""
    ac = _make("tiny", 18, 1)
    _check_against_autograd(ac, 4096, 18, 1, "elu")


def test_actor_and_critic_of_different_shapes():
    """Tails of different shapes run as two launches, each net still right."""
    ac = _make("ragged", 2, 1, critic=[512, 256, 128])
    _check_against_autograd(ac, 4096, 2, 1, "elu")


# ---------------------------------------------------------------------------------------------------------------- fused tails (C ABI)
def _tail_ref(x, W2, b2, W3, b3, Wh, bh, f):
    y2 = f(x.double() @ W2.double().T + b2.double())
    y3 = f(y2 @ W3.double().T + b3.double()) if W3 is not None else None
    out = (y3 if y3 is not None else y2) @ Wh.double().T + bh.double()
    return y2, y3, out


# (K1, n2, n3): every ragged instantiation (N2 tile 64 / 128 / 256, N3 tile 0 / 64 / 128), widths inside the tiles and K1 not a multiple
# of 32 (or of 4: its W2 is read through a padded copy)
TAIL_CASES = [(100, 36, 0), (64, 64, 64), (250, 50, 125), (333, 128, 0), (256, 100, 60), (512, 128, 128), (1024, 250, 0), (510, 256, 64),
              (500, 250, 125),
              # n2 leaves whole 32-column k-blocks of the tile empty: the last W3 boxes lie entirely beyond n2 (zero-filled by TMA)
              (256, 80, 40), (256, 150, 64), (200, 4, 64)]


@pytest.mark.parametrize("name", ["elu", "sigmoid"])
@pytest.mark.parametrize("case", TAIL_CASES, ids=lambda c: "-".join(map(str, c)))
def test_ragged_tail_instantiations_match_fp64(case, name):
    """go1_mlp_tail_forward_grouped on shapes outside scripts/train.py's: a grouped pair (heads 12 and 1) and a single problem (head 5),
    ragged M (the last 64-row block partly filled), against fp64.  sigmoid(0) = 0.5 in the padded columns must add nothing."""
    from go1_b200 import capi
    from activation_test_util import MODULES
    K1, n2, n3 = case
    f = MODULES[name]()
    g = torch.Generator(device="cuda").manual_seed(K1 + n2 + n3)
    R = lambda *s: torch.randn(*s, device="cuda", generator=g)
    for M, heads in ((4096 + 37, (12, 1)), (100, (5,))):
        probs, refs, keep = [], [], []
        for nh in heads:
            xp = R(M, capi.row_pitch(K1)) * 0.5
            x = xp[:, :K1]
            W2, b2 = R(n2, K1) / K1 ** 0.5, R(n2) * 0.1
            W3, b3 = (R(n3, n2) / n2 ** 0.5, R(n3) * 0.1) if n3 else (None, None)
            Wh, bh = R(nh, n3 or n2) / (n3 or n2) ** 0.5, R(nh) * 0.1
            W2p = torch.zeros(n2, capi.row_pitch(K1), device="cuda"); W2p[:, :K1] = W2
            W3p = torch.zeros(n3, capi.row_pitch(n2), device="cuda") if n3 else None
            if n3:
                W3p[:, :n2] = W3
            y2 = torch.full((M, capi.row_pitch(n2)), 7.0, device="cuda")
            y3 = torch.full((M, capi.row_pitch(n3)), 7.0, device="cuda") if n3 else None
            out = torch.full((M, nh), 7.0, device="cuda")
            q = capi.Go1TailProblem()
            q.act_kind = capi.ACTIVATIONS[name]
            q.x, q.ldx, q.W2, q.ldw2, q.b2, q.y2, q.ldy2 = x.data_ptr(), x.stride(0), W2p.data_ptr(), W2p.stride(0), b2.data_ptr(), y2.data_ptr(), y2.stride(0)
            if n3:
                q.W3, q.ldw3, q.b3, q.y3, q.ldy3 = W3p.data_ptr(), W3p.stride(0), b3.data_ptr(), y3.data_ptr(), y3.stride(0)
            q.Wh, q.bh, q.nh, q.out, q.ldout = Wh.data_ptr(), bh.data_ptr(), nh, out.data_ptr(), out.stride(0)
            probs.append(q)
            keep += [xp, W2p, W3p, b2, b3, Wh, bh]
            refs.append(((y2, y3, out), _tail_ref(x, W2, b2, W3, b3, Wh, bh, f)))
        arr = (capi.Go1TailProblem * len(probs))(*probs)
        capi.check(capi.lib().go1_mlp_tail_forward_grouped(arr, len(probs), M, K1, n2, n3, capi.stream_ptr()), "tail")
        torch.cuda.synchronize()
        for (y2, y3, out), (r2, r3, ro) in refs:
            for got, want, width in ((y2, r2, n2), (y3, r3, n3), (out, ro, out.shape[1])):
                if want is None:
                    continue
                want = want.detach()
                scale = float(want.abs().max()) + 1e-6
                assert float((got[:, :width].double() - want).abs().max()) < 6e-3 * scale, (M, width, float((got[:, :width].double() - want).abs().max()), scale)
                # the TMA store of y2 writes whole 16-byte chunks: the row padding up to the next multiple of 4 floats may change
                assert bool((got[:, (width + 3) // 4 * 4:] == 7.0).all()), "stores beyond the width"


@pytest.mark.parametrize("name", ["elu", "sigmoid"])
@pytest.mark.parametrize("shape", ["wide", "narrow", "deep", "ragged", "w36_250"])
def test_fused_tails_match_layer_by_layer(shape, name):
    """ActorCritic.forward_all with the fused tails against the layer-by-layer tensor-core path (M = 100: a partly filled 64-row block)."""
    ac = _make(shape, 2, 1, name, seed=5)
    M = 100
    h, priv = torch.randn(M, K0, device="cuda") * 0.5, torch.randn(M, 2, device="cuda")
    res = {}
    for fuse in (False, True):
        ac.fuse_tail = fuse
        ac.forward_all(h, priv, tag="tailtest%d" % fuse)
        torch.cuda.synchronize()
        res[fuse] = [[t.clone() for t in outs] for outs in (ac._a_out, ac._p_out, ac._c_out)]
    for net in range(3):
        assert len(res[True][net]) == len(res[False][net])
        for a, b in zip(res[False][net], res[True][net]):
            scale = float(a.abs().max()) + 1e-6
            assert float((a - b).abs().max()) < 4e-3 * scale, (net, float((a - b).abs().max()), scale)


# ---------------------------------------------------------------------------------------------------------------- the update's products
# shape, E -> the tails of forward_all + adaptation_forward: {(kernel, N2, K1, N3, head columns, problems)}
UPDATE_CASES = {
    # actor + critic 250-125-head tails grouped in one grid; the adaptation module's 125-head tail
    ("ragged", 2): {("tail3", 250, 500, 125, 12 + 1, 2), ("tail2", 125, 250, 0, 2, 1)},
    # the last two hidden layers 36-20 behind the 64-50 layers; heads on 20 and 25 columns
    ("small_last", 2): {("tail3", 36, 50, 20, 12 + 1, 2), ("tail2", 25, 40, 0, 2, 1)},
    # a 4-wide hidden layer; the 18-wide latent head is too wide for a fused tail (12 at most)
    ("tiny", 18): {("tail3", 4, 256, 64, 12 + 1, 2)},
}


@pytest.mark.parametrize("shape,E", list(UPDATE_CASES), ids=lambda v: str(v))
def test_update_products_on_tensor_cores_with_fused_tails(shape, E, tmp_path, monkeypatch):
    """At gemm_impl = 1 every product of forward_all, backward_ppo and backward_adaptation runs on the wgmma kernels (none on the fp32
    CUDA-core sgemm), the timing CSV lists each of them, and the tails appear as fused launches.  The narrow heads (last hidden width
    below 32, or E = 18 behind a 6-wide layer) are the cases a head's gradient rows are not TMA-readable."""
    from go1_b200 import capi
    out = tmp_path / "gemm.csv"
    monkeypatch.setenv("GO1_GEMM_TIMING_CSV", str(out))
    ac = _make(shape, E, 1)
    M = 4096
    h, priv = torch.randn(M, K0, device="cuda") * 0.3, torch.randn(M, E, device="cuda")
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")
    ac.forward_all(h, priv, tag="train")        # warm (packed copies, buffers)
    L = capi.lib()
    calls = {"gemm1": 0, "gemm0": 0, "grouped": 0, "tail": 0}
    real = {n: getattr(L, n) for n in ("go1_gemm_ex", "go1_gemm_grouped", "go1_mlp_tail_forward_grouped")}

    def gemm_ex(*a):
        calls["gemm%d" % a[12]] += 1
        return real["go1_gemm_ex"](*a)

    def grouped(*a):
        calls["grouped"] += 1
        return real["go1_gemm_grouped"](*a)

    def tail(*a):
        calls["tail"] += 1
        return real["go1_mlp_tail_forward_grouped"](*a)
    monkeypatch.setattr(L, "go1_gemm_ex", gemm_ex)
    monkeypatch.setattr(L, "go1_gemm_grouped", grouped)
    monkeypatch.setattr(L, "go1_mlp_tail_forward_grouped", tail)
    capi.check(L.go1_gemm_timing(1, None, None, None), "timing")
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    outs = ac.adaptation_forward(h)
    ac.backward_adaptation(h, outs, torch.randn(M, E, device="cuda") / M)
    capi.check(L.go1_gemm_timing(0, None, None, None), "timing")
    torch.cuda.synchronize()
    rows = list(csv.DictReader(open(out)))
    assert calls["gemm0"] == 0, calls
    assert len(rows) == calls["gemm1"] + calls["grouped"] + calls["tail"], (len(rows), calls)
    tails = [r for r in rows if r["kernel"].startswith("tail")]
    assert {(r["kernel"], int(r["N"]), int(r["K"]), int(r["n3"]), int(r["heads"]), int(r["problems"])) for r in tails} == UPDATE_CASES[(shape, E)], tails
    assert torch.isfinite(ac.flat_grads).all()


# ---------------------------------------------------------------------------------------------------------------- PPO
def test_graph_replayed_act_equals_eager():
    """PPO.act through its captured CUDA graph gives what the eager launches give, on a ragged shape (packed weight copies, padded
    buffers and the ragged tails inside the graph).  The sampled actions are left out: the capture's warm-up passes draw from the
    action-noise stream."""
    from go1_gym_learn.ppo_cse.ppo import PPO
    N, E = 4096, 2
    ac = _make("ragged", E, 1)
    res = {}
    for graphed in (False, True):
        alg = PPO(ac, device="cuda:0")
        alg.use_cuda_graph = graphed
        alg.init_storage(N, 2, [NOBS], [E], [K0], [NA])
        ac.sample_seed, ac._counter_dev = 7, None
        g = torch.Generator(device="cuda").manual_seed(3)
        obs, priv, hist = torch.empty(N, NOBS, device="cuda"), torch.empty(N, E, device="cuda"), torch.empty(N, K0, device="cuda")
        got = []
        for t in range(3):          # graphed: the first call captures, the later ones replay (same input buffers)
            obs.normal_(generator=g); priv.normal_(generator=g); hist.normal_(generator=g).mul_(0.3)
            alg.act(obs, priv, hist)
            tr = alg.transition
            got.append([tr.values.clone(), tr.action_mean.clone()])
            alg.transition.clear()
        res[graphed] = got
    for a, b in zip(res[False], res[True]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


@pytest.mark.parametrize("impl", [0, 1])
def test_full_ppo_cycle_matches_reference_vectors(impl):
    """act x24 -> process_env_step -> compute_returns -> update on the reference's own vectors (tests/golden/make_golden_hidden.py: actor /
    critic [64, 50, 36, 20], adaptation module [40, 25]).  Tolerances of test_activations_gpu.test_full_ppo_cycle_matches_reference_vectors."""
    from ppo_golden_util import seeded_weights, sample_tensor
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    g = np.load(os.path.join(HERE, "golden", "ppo_hidden.npz"))
    dims = [int(x) for x in g["meta/dims"]]
    N, T, NOBS_, NH, NP, NA_, nl = dims[:7]
    hidden, adapt = dims[7:7 + nl], dims[7 + nl:]
    name = "elu"
    AC_Args.gemm_impl, AC_Args.activation = impl, name
    AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims = hidden, hidden, adapt
    k = 1.0 if impl == 0 else 250.0
    ac = ActorCritic(NOBS_, NP, NH, NA_)
    w = seeded_weights({kk: tuple(v.shape) for kk, v in ac.state_dict().items()})
    ac.load_state_dict({kk: torch.from_numpy(v) for kk, v in w.items()})
    alg = PPO(ac, device="cuda:0")
    alg.init_storage(N, T, [NOBS_], [NP], [NH], [NA_])
    C = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for t in range(T):
        ac.injected_eps = C(g["in/eps"][t])
        alg.act(C(g["in/obs"][t]), C(g["in/priv"][t]), C(g["in/hist"][t]))
        infos = {"env_bins": torch.zeros(N, device="cuda"), "time_outs": torch.zeros(N, dtype=torch.bool, device="cuda")}
        alg.process_env_step(C(g["in/rew"][t]), C(g["in/done"][t]), infos)
    alg.compute_returns(C(g["last/hist"]), C(g["last/priv"]))
    st = alg.storage
    for nm, tol in (("actions", 2e-5), ("values", 2e-5), ("actions_log_prob", 1e-4), ("mu", 2e-5), ("returns", 5e-5), ("advantages", 2e-4)):
        got, want = getattr(st, nm).cpu().numpy(), g[f"{name}/storage/{nm}"]
        assert np.allclose(got, want, rtol=1e-4 * k, atol=tol * k), (nm, np.abs(got - want).max())
    alg.fixed_minibatch_indices = C(g["in/perm"])
    losses = alg.update()
    ref = g[f"{name}/update/losses"]
    kl = 1.0 if impl == 0 else 25.0
    assert abs(losses[0] - ref[0]) < 2e-3 * kl * abs(ref[0]) and abs(losses[1] - ref[1]) < 2e-3 * kl and abs(losses[2] - ref[2]) < 2e-3 * kl * abs(ref[2])
    assert abs(losses[5] - ref[5]) < 2e-3 * kl * abs(ref[5])
    if impl == 0:
        assert abs(alg.learning_rate - float(g[f"{name}/update/learning_rate"])) < 1e-12
    for name_k, v in ac.state_dict().items():
        got, want = sample_tensor(v.cpu().numpy(), stride=3), g[f"{name}/final/{name_k}"]
        if impl == 0:
            assert np.allclose(got[:-2], want[:-2], rtol=0, atol=3e-4), (name_k, np.abs(got[:-2] - want[:-2]).max())
        else:
            d = np.abs(got[:-2] - want[:-2])
            assert np.quantile(d, 0.99) < 4e-3 and d.max() < 4e-2, (name_k, np.quantile(d, 0.99), d.max())
