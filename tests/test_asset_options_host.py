"""Cfg.asset -> Go1AssetOptions (go1_b200.config.asset_config, contact_bodies): the contact-body sets in Isaac Gym body order, the
fixed-base / gravity / armature options and the warnings for the options the compiled Go1 model does not simulate."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _cfg(**asset):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    for k, v in asset.items():
        setattr(Cfg.asset, k, v)
    return Cfg


def test_body_names_are_the_isaac_gym_order():
    from go1_b200.config import BODY_NAMES
    assert len(BODY_NAMES) == 17 and BODY_NAMES[0] == "base"
    assert BODY_NAMES[1:5] == ["FL_hip", "FL_thigh", "FL_calf", "FL_foot"] and BODY_NAMES[13:] == ["RR_hip", "RR_thigh", "RR_calf", "RR_foot"]


def test_train_config_resolves_to_the_sets_the_kernel_used_to_hard_code():
    from go1_b200.config import asset_config, contact_bodies
    b = contact_bodies(_cfg())
    # tests/golden/make_golden.py's penalised_contact_indices / termination_contact_indices / feet_indices
    assert b == dict(penalised=[2, 6, 10, 14, 3, 7, 11, 15], termination=[0], feet=[4, 8, 12, 16])
    o = asset_config(_cfg())
    assert [float(w) for w in o.penalty_weight] == [1.0 if i in (2, 6, 10, 14, 3, 7, 11, 15) else 0.0 for i in range(17)]
    assert o.termination_mask == 1 and o.fix_base == 0 and o.disable_gravity == 0 and o.armature == 0.0


def test_duplicate_selections_add_up():
    from go1_b200.config import BODY_NAMES, asset_config, contact_bodies
    cfg = _cfg(penalize_contacts_on=["thigh", "FL"])
    b = contact_bodies(cfg)
    assert b["penalised"] == [2, 6, 10, 14, 1, 2, 3, 4]                     # extend per entry, as the reference
    w = list(asset_config(cfg).penalty_weight)
    assert w[BODY_NAMES.index("FL_thigh")] == 2.0
    assert w[BODY_NAMES.index("FL_hip")] == 1.0 and w[BODY_NAMES.index("FR_thigh")] == 1.0 and w[BODY_NAMES.index("FR_calf")] == 0.0


def test_termination_bits():
    from go1_b200.config import asset_config
    o = asset_config(_cfg(terminate_after_contacts_on=["base", "thigh"]))
    assert bin(o.termination_mask).count("1") == 5
    assert o.termination_mask == 1 | (1 << 2) | (1 << 6) | (1 << 10) | (1 << 14)
    assert asset_config(_cfg(terminate_after_contacts_on=[])).termination_mask == 0


def test_fixed_base_gravity_and_armature_are_read():
    from go1_b200.config import asset_config
    o = asset_config(_cfg(fix_base_link=True, disable_gravity=True, armature=0.01))
    assert (o.fix_base, o.disable_gravity) == (1, 1) and abs(o.armature - 0.01) < 1e-9


@pytest.mark.parametrize("foot_name", ["None", "calf", "FL_foot", "a"])
def test_bad_foot_name_raises(foot_name):
    from go1_b200.config import asset_config
    with pytest.raises(ValueError, match="foot_name"):
        asset_config(_cfg(foot_name=foot_name))


@pytest.mark.parametrize("armature", [-0.01, float("nan"), float("inf"), "heavy"])
def test_bad_armature_raises(armature):
    from go1_b200.config import asset_config
    with pytest.raises(ValueError, match="armature"):
        asset_config(_cfg(armature=armature))


def test_build_sim_config_returns_the_options():
    from go1_b200.config import build_sim_config
    _, info = build_sim_config(_cfg(fix_base_link=True, penalize_contacts_on=["calf"]), num_envs=8)
    assert info["asset"].fix_base == 1 and info["contact_bodies"]["penalised"] == [3, 7, 11, 15]
    with pytest.raises(ValueError):
        build_sim_config(_cfg(foot_name="toe"), num_envs=8)


@pytest.mark.parametrize("key,value", [("linear_damping", 0.1), ("angular_damping", 0.5), ("max_linear_velocity", 10.),
                                       ("max_angular_velocity", 10.), ("default_dof_drive_mode", 1), ("collapse_fixed_joints", False),
                                       ("file", "{MINI_GYM_ROOT_DIR}/resources/robots/a1/urdf/a1.urdf")])
def test_unsimulated_option_warns_once(capsys, key, value):
    from go1_b200.config import build_sim_config
    build_sim_config(_cfg(**{key: value}), num_envs=8)
    out = capsys.readouterr().out
    lines = [l for l in out.splitlines() if l.startswith("Warning: Cfg.asset.")]
    assert len(lines) == 1 and key in lines[0], out
    if key == "file":
        assert "compiled Go1 model" in lines[0]


def test_documented_no_op_options_do_not_warn(capsys):
    from go1_b200.config import build_sim_config
    build_sim_config(_cfg(density=0.01, thickness=0.02, flip_visual_attachments=True, replace_cylinder_with_capsule=False), num_envs=8)
    assert "Warning: Cfg.asset." not in capsys.readouterr().out
    build_sim_config(_cfg(), num_envs=8)
    assert "Warning: Cfg.asset." not in capsys.readouterr().out


def test_dict_asset_section_from_a_restored_run():
    """scripts/play.py restores Cfg from parameters.pkl; a section may come back as a plain dict."""
    import types
    from go1_b200.config import asset_config
    cfg = types.SimpleNamespace(asset=dict(file="go1.urdf", foot_name="foot", penalize_contacts_on=["thigh", "calf"],
                                           terminate_after_contacts_on=["base"], fix_base_link=False))
    o = asset_config(cfg)
    assert o.termination_mask == 1 and sum(o.penalty_weight) == 8.0


def test_ctypes_mirror_layout():
    import ctypes
    from go1_b200 import capi
    assert ctypes.sizeof(capi.Go1AssetOptions) == 17 * 4 + 4 + 4 + 4 + 4
    assert capi.Go1AssetOptions.armature.offset == 17 * 4 + 12


def test_fixed_base_restatement_conserves_energy():
    """The fp64 restatement used by the GPU tests: M symmetric positive definite, and an unactuated swing under gravity keeps
    kinetic + potential energy to the integrator's O(dt) drift."""
    import numpy as np
    import fixed_base_oracle as fb
    rng = np.random.default_rng(0)
    R0 = fb.quat_to_R([0.1, -0.05, 0.2, 0.97] / np.linalg.norm([0.1, -0.05, 0.2, 0.97]))
    q = np.tile([0.1, 0.8, -1.5], 4) + rng.uniform(-0.3, 0.3, 12)
    qd = rng.uniform(-2, 2, 12)
    for leg in range(4):
        M = np.stack([fb.rnea(leg, R0, q[3 * leg:3 * leg + 3], np.zeros(3), e, np.zeros(3)) for e in np.eye(3)], 1)
        assert np.allclose(M, M.T, atol=1e-12) and np.linalg.eigvalsh(M).min() > 0
    g = [0.0, 0.0, -9.81]
    e0 = fb.energy(R0, q, qd, g)
    q1, qd1 = fb.policy_step(R0, q, qd, lambda q, qd: np.zeros(12), g, 2e-5, 800)
    assert abs(fb.energy(R0, q1, qd1, g) - e0) < 2e-3 * max(abs(e0), 1.0)
    assert np.abs(q1 - q).max() > 1e-3                       # it did swing
