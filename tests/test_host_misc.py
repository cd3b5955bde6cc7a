"""Host-side pieces that need no GPU: the category generator shared with the device kernel, the lazy extras containers, the
bench.py reference arm's JSON contract."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "walk-these-ways_b200"), os.path.join(ROOT, "walk-these-ways_b200", "compat")]


def test_splitmix64_stream_is_chunking_invariant_and_matches_the_scalar_recurrence():
    from go1_b200.curriculum_dev import SplitMix64
    a, b = SplitMix64(101), SplitMix64(101)
    x = a.random(37)
    y = np.concatenate([b.random(k) for k in (1, 5, 0, 20, 11)])
    assert np.array_equal(x, y) and a.state == b.state          # the device kernel draws one value at a time
    # scalar restatement with Python integers (the CUDA code of csrc/curriculum.cu::splitmix_next)
    M, st, out = (1 << 64) - 1, 101, []
    for _ in range(37):
        st = (st + 0x9E3779B97F4A7C15) & M
        z = st
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        z ^= z >> 31
        out.append((z >> 11) / 9007199254740992.0)
    assert np.array_equal(x, np.array(out)) and st == a.state
    assert 0.0 <= x.min() and x.max() < 1.0 and abs(SplitMix64(7).random(20000).mean() - 0.5) < 0.01


def test_lazy_containers_build_once_and_pickle_as_plain_dicts():
    from go1_gym.envs.base.legged_robot import LazyExtras, _LazyDict
    calls = []
    d = _LazyDict(lambda: calls.append(1) or {"a": 1, "b": np.arange(3)})
    assert calls == []
    assert "a" in d and len(d) == 2 and calls == [1] and d["a"] == 1 and calls == [1]
    back = pickle.loads(pickle.dumps(_LazyDict(lambda: {"w": np.ones(2)})))
    assert type(back) is dict and np.array_equal(back["w"], np.ones(2))
    ex = LazyExtras()
    n = []
    ex.lazy("joint_pos", lambda: n.append(1) or "fresh")
    assert "joint_pos" in ex and ex["joint_pos"] == "fresh" and ex.get("joint_pos") == "fresh" and len(n) == 2     # evaluated per read
    assert ex.get("missing", 3) == 3


def test_bench_reference_arm_prints_the_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1", "--cpu-envs", "8"],
                         capture_output=True, text=True, timeout=600, env={**os.environ, "RANK": "0"})
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "env_steps_per_s" and line["unit"] == "env-steps/s" and line["higher_is_better"] is True
    assert line["value"] > 0 and line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"] == {"value": line["value"], "unit": line["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # the same workload definition as the GPU arm prints (the bounded sample is named separately), fixed thread count <= 32
    assert line["config"]["name"] == "flat" and line["config"]["envs_per_gpu"] == 4096 and line["scaling"] == "weak" and line["warmup"] == 1
    assert "8 envs x 24-step rollout" in line["sample"] and line["cpu_baseline"]["cores"] <= 32
    # other ranks of a torchrun launch do no work and print nothing
    out1 = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1"], capture_output=True, text=True,
                          timeout=120, env={**os.environ, "RANK": "1"})
    assert out1.returncode == 0 and out1.stdout.strip() == ""
