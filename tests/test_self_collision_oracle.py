"""The self-collision model (DESIGN.md §3) in the fp64 oracle: no contact at nominal poses, contacts of crossed legs that conserve
momentum and gain no energy, bounded penetration, reported base and foot forces, and the Python side of the switch."""
import ctypes as C

import numpy as np

import self_collision_oracle as so
from oracle import physics as ph

P = so.DEFAULTS
D = ph.DEFAULT_DOF_POS
FEET = [4, 8, 12, 16]


def _free_params():
    pp = ph.default_params()
    pp.gravity[2] = 0.0
    return pp


def test_nominal_poses_have_no_self_contact_and_match_the_switch_off_oracle():
    rng = np.random.default_rng(0)
    pp = ph.default_params()
    for i in range(200):
        q = D + rng.uniform(-0.1, 0.1, 12)
        args = ([0, 0, 0.3 + rng.uniform(0, 0.05)], [0, 0, 0, 1], rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.3, 0.3, 3), q, rng.uniform(-1, 1, 12))
        tau, cf, hits, _ = so.self_forces(*args, 1.0, P)
        assert hits == 0 and not tau.any() and not cf.any()
        a, b = ph.make_state(*args), ph.make_state(*args)
        t = rng.uniform(-5, 5, 12)
        ca, _ = so.substep(pp, ph.make_dr(), a, t, P)
        cb = ph.substep(pp, ph.make_dr(), b, t)
        assert np.array_equal(ca, cb)
        for k in ("pos", "quat", "linvel", "angvel", "q", "qd"):
            assert np.array_equal(np.array(getattr(a, k)), np.array(getattr(b, k))), k


def _crossed(seed):
    """Front legs adducted towards each other and rear legs swung under the body, approaching at a few rad/s."""
    rng = np.random.default_rng(seed)
    q = D.copy()
    q[0], q[3] = -0.3 + rng.uniform(-0.05, 0.05), 0.3 + rng.uniform(-0.05, 0.05)
    q[6], q[9] = -0.3 + rng.uniform(-0.05, 0.05), 0.3 + rng.uniform(-0.05, 0.05)
    qd = np.zeros(12)
    qd[0], qd[3], qd[6], qd[9] = -3.0, 3.0, -3.0, 3.0
    qd += rng.uniform(-0.5, 0.5, 12)
    return ph.make_state([0, 0, 2.0], [0, 0, 0, 1], rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.2, 0.2, 3), q, qd)


def test_crossed_legs_collide_and_conserve_momentum_in_free_flight():
    """Self contacts add no more momentum drift than the bound test_momentum_conserved_under_internal_torques allows the
    integrator (1e-3 linear, 3e-3 angular) to the drift of the same motion without them."""
    from test_physics_oracle import momentum_energy
    pp = _free_params()
    for seed in range(3):
        drift = []
        for model in (None, P):
            s = _crossed(seed)
            P0, L0, _, _ = momentum_energy(s)
            hits = 0
            for _ in range(100):
                hits += so.substep(pp, ph.make_dr(), s, np.zeros(12), model)[1]
            P1, L1, _, _ = momentum_energy(s)
            drift.append((np.abs(P1 - P0).max(), np.abs(L1 - L0).max(), hits))
            assert all(np.isfinite(np.array(getattr(s, k))).all() for k in ("pos", "quat", "linvel", "angvel", "q", "qd"))
        (p_off, l_off, _), (p_on, l_on, hits) = drift
        assert hits > 0
        assert p_on <= p_off + 1e-3 and l_on <= l_off + 3e-3, drift


def test_pressed_calves_stay_shallow_and_finite():
    """Front calves driven into each other by opposing 1 N m hip torques for 1 s (200 substeps): penetration below 5 mm."""
    pp = _free_params()
    q = D.copy(); q[0], q[3] = -0.3, 0.3
    s = ph.make_state([0, 0, 2.0], [0, 0, 0, 1], [0, 0, 0], [0, 0, 0], q, np.zeros(12))
    tau = np.zeros(12); tau[0], tau[3] = -1.0, 1.0
    deepest, hits = 0.0, 0
    for _ in range(200):
        deepest = max(deepest, so.self_forces(s.pos, s.quat, s.linvel, s.angvel, s.q, s.qd, 1.0, P)[3])
        _, h = so.substep(pp, ph.make_dr(), s, tau, P)
        hits += h
    assert hits > 20
    assert deepest < 5e-3, deepest
    assert all(np.isfinite(np.array(getattr(s, k))).all() for k in ("pos", "quat", "linvel", "angvel", "q", "qd"))


def test_free_flight_contacts_gain_no_energy():
    """Kinetic energy (no gravity, no torques) after 100 substeps of crossed-leg contacts does not exceed the start by more than
    the 2 % the drop test allows."""
    pp = _free_params()
    for seed in range(3):
        s = _crossed(seed)
        e0 = energy(s)
        for _ in range(100):
            so.substep(pp, ph.make_dr(), s, np.zeros(12), P)
        assert energy(s) <= 1.02 * e0 + 1e-9, (e0, energy(s))


def energy(s):
    """Kinetic energy of the articulation (the T of test_physics_oracle.momentum_energy)."""
    from test_physics_oracle import momentum_energy
    return momentum_energy(s)[2]


def test_knee_into_trunk_reports_base_force_and_feet_report_both_rows():
    # FL hip rolled under the body (-2.62 rad) with the thigh at 1.18 rad: the knee presses into the trunk from below.  The base row
    # reports the reaction of the knee probe, which acts on the thigh body
    q = D.copy(); q[0], q[1], q[2] = -2.6166666666666667, 1.1775, -2.7
    tau, cf, hits, _ = so.self_forces([0, 0, 1], [0, 0, 0, 1], [0, 0, 0], [0, 0, 0], q, np.zeros(12), 1.0, P)
    assert np.linalg.norm(cf[0]) > 1.0 and np.allclose(cf[0], -cf[2]) and not cf[3].any() and not cf[4].any()
    # both front feet at one point (nearly): each foot row carries the contact, with opposite signs
    q = D.copy()
    for qh in np.linspace(-0.2, -0.6, 81):
        q[0], q[3] = qh, -qh + 0.002
        tau, cf, hits, _ = so.self_forces([0, 0, 1], [0, 0, 0, 1], [0, 0, 0], [0, 0, 0], q, np.zeros(12), 1.0, P)
        if np.linalg.norm(cf[FEET[0]]) > 0 and np.linalg.norm(cf[FEET[1]]) > 0:
            break
    assert np.linalg.norm(cf[FEET[0]]) > 0 and np.linalg.norm(cf[FEET[1]]) > 0
    assert np.allclose(cf[FEET[0]] + cf[FEET[1]] + cf[2] + cf[3] + cf[6] + cf[7] + cf[0], 0.0, atol=1e-9)


def test_switch_resolution_and_ctypes_mirror():
    import os
    from go1_b200 import capi
    from go1_b200.config import self_collision_config
    lib = C.CDLL(capi.LIB_PATH)
    assert lib.go1_sizeof_self_collision() == C.sizeof(capi.Go1SelfCollision)

    class Asset:
        self_collisions = 0

    class Cfg:
        asset = Asset
    Asset.model_self_collisions = True
    assert self_collision_config(Cfg).enabled == 1
    Asset.self_collisions = 1                      # the reference's "1 to disable"
    assert self_collision_config(Cfg).enabled == 0
    Asset.self_collisions = 0
    Asset.model_self_collisions = False
    assert self_collision_config(Cfg).enabled == 0
    del Asset.model_self_collisions                # a restored parameters.pkl without the key: the environment switch decides
    old = os.environ.pop("GO1_SELF_COLLISIONS", None)
    try:
        assert self_collision_config(Cfg).enabled == 0
        os.environ["GO1_SELF_COLLISIONS"] = "1"
        assert self_collision_config(Cfg).enabled == 1
    finally:
        os.environ.pop("GO1_SELF_COLLISIONS", None)
        if old is not None:
            os.environ["GO1_SELF_COLLISIONS"] = old
