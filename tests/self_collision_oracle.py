"""fp64 restatement of the self-collision model of the step kernel (DESIGN.md §3) on top of the physics oracle.

Geometry: thigh capsule from the thigh joint p1 to the knee p2, calf capsule from p2 to the foot point pf, foot sphere at pf, trunk
box GO1_BASE_BOX_HALF about the base origin.  Pairs: thigh/calf/foot of a leg against thigh/calf/foot of every other leg, and each
leg's knee, calf midpoint and foot as spheres against the trunk.  Penalty law: fn = max(k depth - c v_n, 0), friction
min(mu fn / |v_t|, pen_mt / dt) along -v_t with mu = the env's robot friction.

Every self-contact force acts on two bodies of the same robot with equal and opposite forces at one point, so its generalised
force has no base component: it enters the oracle substep exactly as the joint torques J^T F of the two bodies.  The kernel
instead applies the spatial forces in its articulated-body pass; the two routes agree up to rounding.  The forces are added to
the reported rows (Isaac Gym body order: base, then hip, thigh, calf, foot per leg).
"""
import os
import re

import numpy as np

from oracle import physics as ph

_HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "walk-these-ways_b200", "csrc", "go1_model_generated.h")


def _model():
    txt = open(_HDR).read()
    arr = lambda name: np.array([float(x) for x in re.search(name + r"\[[^=]*=\s*\{([^}]*)\}", txt).group(1).split(",")])
    return dict(hip=arr("GO1_HIP_ORIGIN").reshape(4, 3), thigh=arr("GO1_THIGH_ORIGIN").reshape(4, 3), calf=arr("GO1_CALF_ORIGIN").reshape(4, 3),
                foot=arr("GO1_FOOT_OFFSET").reshape(4, 3), box=arr("GO1_BASE_BOX_HALF"))


M = _model()
DEFAULTS = dict(k=5000.0, c=20.0, thigh_radius=0.017, calf_radius=0.008, foot_radius=0.02)


def quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _axis_R(axis, q):
    c, s = np.cos(q), np.sin(q)
    if axis == 0:
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def kinematics(pos, quat, linvel, angvel, q, qd):
    """Per leg: joint origins p0, p1, p2 and foot pf, world joint axes, world angular velocities and origin velocities of the
    hip, thigh and calf bodies."""
    pos, linvel, angvel, q, qd = (np.asarray(a, dtype=np.float64) for a in (pos, linvel, angvel, q, qd))
    R0 = quat_to_R(np.asarray(quat, dtype=np.float64))
    legs = []
    for L in range(4):
        Rw0 = R0 @ _axis_R(0, q[3 * L]); Rw1 = Rw0 @ _axis_R(1, q[3 * L + 1]); Rw2 = Rw1 @ _axis_R(1, q[3 * L + 2])
        p0 = pos + R0 @ M["hip"][L]; p1 = p0 + Rw0 @ M["thigh"][L]; p2 = p1 + Rw1 @ M["calf"][L]; pf = p2 + Rw2 @ M["foot"][L]
        ax = [Rw0[:, 0], Rw1[:, 1], Rw2[:, 1]]
        w0 = angvel + ax[0] * qd[3 * L]; w1 = w0 + ax[1] * qd[3 * L + 1]; w2 = w1 + ax[2] * qd[3 * L + 2]
        v0 = linvel + np.cross(angvel, p0 - pos); v1 = v0 + np.cross(w0, p1 - p0); v2 = v1 + np.cross(w1, p2 - p1)
        legs.append(dict(p=[p0, p1, p2], pf=pf, ax=ax, w=[w0, w1, w2], v=[v0, v1, v2]))
    return R0, legs


def closest_segments(p0, p1, q0, q1):
    d1, d2, r = p1 - p0, q1 - q0, p0 - q0
    a, e, f = d1 @ d1, d2 @ d2, d2 @ r
    s = t = 0.0
    cl = lambda x: min(max(x, 0.0), 1.0)
    if a > 0 and e > 0:
        b, c = d1 @ d2, d1 @ r
        den = a * e - b * b
        s = cl((b * f - c * e) / den) if den > 1e-6 * a * e else 0.0
        t = (b * s + f) / e
        if t < 0:
            t, s = 0.0, cl(-c / a)
        elif t > 1:
            t, s = 1.0, cl((b - c) / a)
    elif a > 0:
        s = cl(-(d1 @ r) / a)
    elif e > 0:
        t = cl(f / e)
    return p0 + s * d1, q0 + t * d2


def _force(P, n, depth, vrel, mu, pen_mt_dt):
    vn = vrel @ n
    fn = max(P["k"] * depth - P["c"] * vn, 0.0)
    vt = vrel - vn * n
    vtn = np.sqrt(vt @ vt)
    ct = min(mu * fn / vtn, pen_mt_dt) if vtn > 1e-9 else 0.0
    return fn * n - ct * vt


def self_forces(pos, quat, linvel, angvel, q, qd, friction, P, pen_mt_dt=0.2 / 0.005):
    """(tau_self [12], contact rows [17][3], number of touching shape pairs, deepest penetration) of one robot state."""
    R0, legs = kinematics(pos, quat, linvel, angvel, q, qd)
    pos, linvel, angvel = (np.asarray(a, dtype=np.float64) for a in (pos, linvel, angvel))
    rad = [P["thigh_radius"], P["calf_radius"], P["foot_radius"]]
    tau = np.zeros(12)
    cf = np.zeros((17, 3))
    hits, deepest = 0, 0.0

    def seg(g, k):
        return (g["p"][1], g["p"][2]) if k == 0 else ((g["p"][2], g["pf"]) if k == 1 else (g["pf"], g["pf"]))

    def vel(g, k, x):
        b = 1 if k == 0 else 2
        return g["v"][b] + np.cross(g["w"][b], x - g["p"][b])

    def apply(L, k, x, F):
        nj = 2 if k == 0 else 3                  # the thigh is moved by joints 0-1, the calf and foot by 0-2
        for j in range(nj):
            tau[3 * L + j] += legs[L]["ax"][j] @ np.cross(x - legs[L]["p"][j], F)
        cf[2 + k + 4 * L] += F

    for A in range(4):
        for B in range(A + 1, 4):
            for i in range(3):
                for j in range(3):
                    c1, c2 = closest_segments(*seg(legs[A], i), *seg(legs[B], j))
                    dl = c2 - c1
                    d2, rs = dl @ dl, rad[i] + rad[j]
                    if d2 < rs * rs and d2 > 1e-12:
                        dist = np.sqrt(d2)
                        n = dl / dist
                        depth = rs - dist
                        x = c1 + (rad[i] - 0.5 * depth) * n
                        Fb = _force(P, n, depth, vel(legs[B], j, x) - vel(legs[A], i, x), friction, pen_mt_dt)
                        apply(A, i, x, -Fb)
                        apply(B, j, x, Fb)
                        hits += 1
                        deepest = max(deepest, depth)
    h = M["box"]
    for L in range(4):
        g = legs[L]
        for k, c in enumerate((g["p"][2], 0.5 * (g["p"][2] + g["pf"]), g["pf"])):
            r = rad[k]
            lc = R0.T @ (c - pos)
            dl = lc - np.clip(lc, -h, h)
            d2 = dl @ dl
            if d2 >= r * r:
                continue
            if d2 > 0:
                dist = np.sqrt(d2)
                nl, depth = dl / dist, r - dist
            else:
                e = h - np.abs(lc)
                a = int(np.argmin(e))
                nl = np.zeros(3); nl[a] = -1.0 if lc[a] < 0 else 1.0
                depth = r + e[a]
            n = R0 @ nl
            x = c - (r - 0.5 * depth) * n
            Fl = _force(P, n, depth, vel(g, k, x) - (linvel + np.cross(angvel, x - pos)), friction, pen_mt_dt)
            apply(L, k, x, Fl)
            cf[0] -= Fl
            hits += 1
            deepest = max(deepest, depth)
    return tau, cf, hits, deepest


def substep(pp, dr, s, tau, P):
    """One oracle substep with the self-collision model P (None = off).  Returns the contact rows [17][3] and the pair count."""
    if P is None:
        return ph.substep(pp, dr, s, tau), 0
    ts, cs, hits, _ = self_forces(s.pos, s.quat, s.linvel, s.angvel, s.q, s.qd, dr.friction, P, pp.pen_mt / pp.dt)
    cf = ph.substep(pp, dr, s, np.asarray(tau, dtype=np.float64) + ts)
    return cf + cs, hits
