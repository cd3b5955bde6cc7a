"""fp64 restatement of a Go1 leg on a welded base (Cfg.asset.fix_base_link, DESIGN.md §3), from resources/go1_model.json.

With the base fixed each leg is an independent 3-DOF chain (hip about x, thigh and calf about y), so its dynamics is the
joint-space equation

    (M(q) + armature I) q'' = tau - C(q, q') q' - g(q)

with M, C q' + g evaluated by the recursive Newton-Euler algorithm in world coordinates: C q' + g = RNEA(q, q', 0) with the base
accelerating at -a_g (0 with gravity off), column i of M = RNEA(q, 0, e_i) without gravity.  No contacts (the feet hang free) and
no joint-limit terms (the joints stay inside their limits).  Integration is the step kernel's semi-implicit Euler per substep:
q' += dt q'', q += dt q'.
"""
import json
import os

import numpy as np

_JSON = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "walk-these-ways_b200", "resources", "go1_model.json")
MODEL = json.load(open(_JSON))
PARTS = ("hip", "thigh", "calf")


def rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    if axis == 0:
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def rnea(leg, R0, q, qd, qdd, a_base):
    """Joint torques of leg `leg` for (q, q', q'') on a base with orientation R0 whose origin accelerates at a_base (world)."""
    o, R = np.zeros(3), R0
    w, al, acc = np.zeros(3), np.zeros(3), np.array(a_base, dtype=np.float64)
    links = []
    for j, part in enumerate(PARTS):
        d = MODEL[part][leg]
        r = R @ np.array(d["origin"])                  # joint origin relative to the parent's origin
        acc = acc + np.cross(al, r) + np.cross(w, np.cross(w, r))
        o = o + r
        R = R @ rot(d["axis"], q[j])
        ax = R[:, d["axis"]]
        w_new = w + ax * qd[j]
        al = al + ax * qdd[j] + np.cross(w, ax * qd[j])
        w = w_new
        c = R @ np.array(d["com"])
        ac = acc + np.cross(al, c) + np.cross(w, np.cross(w, c))
        I = R @ np.array(d["inertia_com"]) @ R.T
        f = d["mass"] * ac
        n = I @ al + np.cross(w, I @ w)
        links.append((o.copy(), c, ax, f, n))
    tau = np.zeros(3)
    F, N, o_next = np.zeros(3), np.zeros(3), None
    for j in (2, 1, 0):
        o_j, c, ax, f, n = links[j]
        N = n + np.cross(c, f) + N + (np.cross(o_next - o_j, F) if o_next is not None else 0.0)
        F = f + F
        tau[j] = ax @ N
        o_next = o_j
    return tau


def joint_accel(leg, R0, q, qd, tau, gravity, armature=0.0):
    """q'' of one leg on a welded base: (M + armature I)^-1 (tau - C q' - g)."""
    g = np.asarray(gravity, dtype=np.float64)
    bias = rnea(leg, R0, q, qd, np.zeros(3), -g)
    M = np.stack([rnea(leg, R0, q, np.zeros(3), e, np.zeros(3)) for e in np.eye(3)], 1)
    return np.linalg.solve(M + armature * np.eye(3), tau - bias)


def policy_step(R0, q, qd, torque_fn, gravity, dt, decimation, armature=0.0):
    """`decimation` substeps of all four legs: q, q' [12] -> new q, q'.  torque_fn(q, q') -> tau [12] per substep."""
    q, qd = np.array(q, dtype=np.float64), np.array(qd, dtype=np.float64)
    for _ in range(decimation):
        tau = torque_fn(q, qd)
        for leg in range(4):
            s = slice(3 * leg, 3 * leg + 3)
            qdd = joint_accel(leg, R0, q[s], qd[s], tau[s], gravity, armature)
            qd[s] = qd[s] + dt * qdd
            q[s] = q[s] + dt * qd[s]
    return q, qd


def energy(R0, q, qd, gravity):
    """Kinetic + potential energy of the four legs (base welded at the origin): a check of the restatement."""
    g = np.asarray(gravity, dtype=np.float64)
    e = 0.0
    for leg in range(4):
        s = slice(3 * leg, 3 * leg + 3)
        M = np.stack([rnea(leg, R0, q[s], np.zeros(3), col, np.zeros(3)) for col in np.eye(3)], 1)
        e += 0.5 * qd[s] @ M @ qd[s]
        o, R = np.zeros(3), R0
        for j, part in enumerate(PARTS):
            d = MODEL[part][leg]
            o = o + R @ np.array(d["origin"])
            R = R @ rot(d["axis"], q[s][j])
            e -= d["mass"] * g @ (o + R @ np.array(d["com"]))
    return e
