"""The learner's launch trace: every call of a go1_* entry point that capi.lib() binds, in call order, with every argument.

Pointers into ActorCritic.flat_params / flat_grads are recorded as ["P" | "G", offset in floats]; any other device pointer as "S<n>",
numbered by its first appearance in the case, and streams likewise as "T<n>", so the trace shows which buffers and which of the two
streams each launch uses without depending on where the allocator put them.  Structures (Go1GemmEpilogue, which _Net reuses between
calls, Go1TailProblem, Go1CopySeg, Go1Bf16Seg) are recorded field by field at call time, arrays of them and of pointers element by
element.  Torch-side operations (copy_, fill_, zero_) do not appear; the gradient-parity tests check those.

tests/golden/make_golden_launches.py writes the traces of CASES to tests/golden/launches.json.gz; tests/test_learner_launches_gpu.py
replays them against it."""
import ctypes as C
import gc
import gzip
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in ("walk-these-ways_b200", os.path.join("walk-these-ways_b200", "compat")):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), _p))
FIXTURE = os.path.join(HERE, "golden", "launches.json.gz")

# actor = critic hidden dims, adaptation module hidden dims, and the E the shape is run with (None: any)
SHAPES = {
    "512-256-128": ([512, 256, 128], [256, 128], None),
    "256": ([256], [64], None),
    "64-50-36-20": ([64, 50, 36, 20], [40, 25], None),
    "256-4-64": ([256, 4, 64], [128, 6], 18),
    "130-70-33": ([130, 70, 33], [70, 33], None),
}
MODES = {"impl0": (0, False), "impl1": (1, False), "impl2": (2, False), "impl2b": (2, True)}


def _cases():
    """Every mode meets every shape (and, across its cases, each E in 2 / 5 / 45, each K0 and each M); four more cases per mode vary
    the other parameters on the shapes most of the routes branch on."""
    cases = {}
    shapes = list(SHAPES)
    for mi, mode in enumerate(MODES):
        combos = [(si, si + mi) for si in range(len(shapes))] + [(0, mi + 1), (2, mi + 2), (3, mi + 1), (4, mi + 3)]
        for si, k in combos:
            shape = shapes[si]
            E = SHAPES[shape][2] or (2, 5, 45)[k % 3]
            K0 = (2100, 2130)[k % 2]
            M = (48, 4096)[(si + k // 2) % 2]
            act = ("elu", "tanh")[(k // 3) % 2]
            name = f"{mode}-{shape}-E{E}-K{K0}-M{M}-{act}"
            cases[name] = dict(mode=mode, shape=shape, E=E, K0=K0, M=M, act=act)
        cases[f"{mode}-ppo-cycle"] = dict(mode=mode, shape="512-256-128", E=2, K0=2100, M=None, act="elu")
    return cases


CASES = _cases()


class Tracer:
    """Wraps every go1_* function of capi.lib() (setattr on the CDLL) and appends one record per call to self.calls."""

    def __init__(self, ac):
        self.ac, self.calls, self.labels, self.streams = ac, [], {}, {}

    def _ptr(self, v):
        if isinstance(v, C.c_void_p):
            v = v.value
        if v is None:
            return None
        for tag, buf in (("P", self.ac._flat), ("G", self.ac._grad)):
            if buf is not None and buf.data_ptr() <= v < buf.data_ptr() + 4 * buf.numel():
                return [tag, (v - buf.data_ptr()) // 4]
        return self.labels.setdefault(v, "S%d" % len(self.labels))

    def _stream(self, v):
        v = v.value if isinstance(v, C.c_void_p) else v
        return self.streams.setdefault(v, "T%d" % len(self.streams))

    def _struct(self, s):
        return [self._ptr(getattr(s, f)) if t is C.c_void_p else getattr(s, f) for f, t in s._fields_]

    def _arg(self, t, a):
        if t is C.c_void_p and not isinstance(a, C.Array):
            return self._ptr(a)
        if t in (C.c_void_p, C.POINTER(C.c_void_p)):
            return [self._ptr(x) for x in a]
        if isinstance(t, type) and issubclass(t, C._Pointer):
            if a is None:
                return None
            if issubclass(t._type_, C.Structure):
                return [self._struct(x) for x in a] if isinstance(a, C.Array) else self._struct(a)
            return "host"
        return a.value if isinstance(a, C._SimpleCData) else a

    def install(self, monkeypatch):
        from go1_b200 import capi
        L = capi.lib()
        for name, fn in list(vars(L).items()):
            if not name.startswith("go1_") or not fn.argtypes:
                continue
            types = list(fn.argtypes)
            stream_last = types[-1] is C.c_void_p

            def call(*args, _fn=fn, _name=name, _types=types, _stream_last=stream_last):
                n = len(args) - 1 if _stream_last else len(args)
                rec = [self._arg(t, a) for t, a in zip(_types[:n], args[:n])]
                if _stream_last:
                    rec.append(self._stream(args[-1]))
                self.calls.append([_name, rec])
                return _fn(*args)
            monkeypatch.setattr(L, name, call)


class _Patch:
    """A minimal monkeypatch for the fixture generator (pytest's is used in the test)."""

    def __init__(self):
        self.saved = []

    def setattr(self, obj, name, value):
        self.saved.append((obj, name, getattr(obj, name)))
        setattr(obj, name, value)

    def undo(self):
        for obj, name, value in reversed(self.saved):
            setattr(obj, name, value)
        self.saved = []


def _kmajor(h, priv, out):
    from go1_gym_learn.ppo_cse import actor_critic
    # (commits before history_kmajor took BF16 buffers had a separate history_kmajor_bf16; this lets the generator run there)
    f = getattr(actor_critic, "history_kmajor_bf16", None) if out.dtype == torch.bfloat16 else None
    return (f or actor_critic.history_kmajor)(h, priv, out)


def _learner_case(c, monkeypatch):
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse import ActorCritic
    hidden, adapt, _ = SHAPES[c["shape"]]
    E, K0, M = c["E"], c["K0"], c["M"]
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.actor_hidden_dims = AC_Args.critic_hidden_dims = hidden
    AC_Args.adaptation_module_branch_hidden_dims = adapt
    AC_Args.activation = c["act"]
    torch.manual_seed(0)
    ac = ActorCritic(70, E, K0, 12).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    h = torch.randn(M, capi.history_pitch(K0), device="cuda", generator=g)[:, :K0]
    priv = torch.randn(M, E, device="cuda", generator=g)
    dmean = torch.randn(M, 12, device="cuda", generator=g) / M
    dvalue = torch.randn(M, 1, device="cuda", generator=g) / M
    dstd = torch.randn(12, device="cuda", generator=g)
    dpred = torch.randn(M, E, device="cuda", generator=g) / M
    if AC_Args.gemm_impl == 2:      # the caller-built hT of RolloutStorage's BF16 minibatches
        hc = torch.empty(M, capi.bf16_pitch(K0), device="cuda", dtype=torch.bfloat16)[:, :K0].copy_(h)
        hT = torch.empty(K0 + 1 + 2 * E, capi.bf16_pitch(M), device="cuda", dtype=torch.bfloat16)
    else:
        hc, hT = h, torch.empty(K0 + 1 + 2 * E, (M + 31) // 32 * 32, device="cuda")
    tracer = Tracer(ac)
    tracer.install(monkeypatch)
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    ac.forward_all(hc, priv, tag="train")
    ac.backward_ppo(hc, priv, dmean, dvalue, dstd, hT=_kmajor(hc, priv, hT))
    outs = ac.adaptation_forward(h)
    ac.backward_adaptation(h, outs, dpred)
    ac.act_student(h)
    ac.act_teacher(h, priv)
    ac.evaluate(h, priv)
    ac.weights_version += 1
    ac.ensure_packed()
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    torch.cuda.synchronize()
    return tracer.calls


def _ppo_case(c, monkeypatch, N=512, T=24):
    """One rollout of random transitions and one PPO update (4 minibatches of N T / 4 rows, 5 epochs), as
    test_bf16_backward_gpu._ppo_cycle: RolloutStorage's minibatches and their hT."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    NOBS, NH, NP, NA = 70, c["K0"], c["E"], 12
    torch.manual_seed(0)
    ac = ActorCritic(NOBS, NP, NH, NA)
    tracer = Tracer(ac)
    tracer.install(monkeypatch)
    alg = PPO(ac, device="cuda:0")
    alg.init_storage(N, T, [NOBS], [NP], [NH], [NA])
    g = torch.Generator(device="cuda").manual_seed(5)
    inputs = []     # every step's inputs stay alive, so that no step's input reuses an earlier step's block
    for t in range(T):
        ac.injected_eps = torch.randn(N, NA, device="cuda", generator=g)
        inputs.append((ac.injected_eps, torch.randn(N, NOBS, device="cuda", generator=g), torch.randn(N, NP, device="cuda", generator=g),
                       torch.randn(N, NH, device="cuda", generator=g), torch.randn(N, device="cuda", generator=g),
                       torch.zeros(N, dtype=torch.bool, device="cuda"), torch.zeros(N, device="cuda"), torch.zeros(N, dtype=torch.bool, device="cuda")))
        _, obs, priv, hist, rew, dones, bins, touts = inputs[-1]
        alg.act(obs, priv, hist)
        alg.process_env_step(rew, dones, {"env_bins": bins, "time_outs": touts})
    alg.compute_returns(torch.randn(N, NH, device="cuda", generator=g), torch.randn(N, NP, device="cuda", generator=g))
    alg.fixed_minibatch_indices = torch.randperm(N * T, device="cuda", generator=g)
    alg.update()
    torch.cuda.synchronize()
    return tracer.calls


def trace(name, monkeypatch):
    """The launch trace of CASES[name] from a fresh ActorCritic, as JSON data; AC_Args is restored afterwards."""
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    c = CASES[name]
    fields = ("gemm_impl", "bf16_backward", "actor_hidden_dims", "critic_hidden_dims", "adaptation_module_branch_hidden_dims", "activation")
    saved = {f: getattr(AC_Args, f) for f in fields}
    AC_Args.gemm_impl, AC_Args.bf16_backward = MODES[c["mode"]]
    # a memory pool of the case's own, and no cyclic garbage collection during the case: which freed block a new buffer reuses (and so
    # which labels two buffers share) then depends on the case alone, not on what ran before it in the process
    pool = torch.cuda.MemPool()
    gc.collect()
    gc.disable()
    try:
        with torch.cuda.use_mem_pool(pool):
            calls = _ppo_case(c, monkeypatch) if c["M"] is None else _learner_case(c, monkeypatch)
            torch.cuda.synchronize()
    finally:
        gc.enable()
        monkeypatch.undo()
        for f, v in saved.items():
            setattr(AC_Args, f, v)
    return json.loads(json.dumps(calls))


def load():
    with gzip.open(FIXTURE, "rt") as f:
        return json.load(f)


def write(commit, traces):
    with open(FIXTURE, "wb") as raw, gzip.GzipFile(fileobj=raw, mode="wb", mtime=0) as f:
        f.write(json.dumps({"commit": commit, "cases": traces}, separators=(",", ":")).encode())
