"""Float64 reference of the tank motion (DESIGN.md section 2.15; sphk_tank_* in sphk.h): the schedule {theta, thd, thdd, R (G - a_w),
a_w} at a time t, written from its definition (theta as a function, its derivatives by the product rule and the spin by its
integral), and one step of the fluid velocities in the tank frame.  numpy only.

A motion is a dict of capi.tank_motion's keys: axis, pivot, roll_amplitude, roll_omega, roll_phase, spin, accel, harmonics
[{amplitude, omega, phase}], ramp.
"""
import numpy as np


def _f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def params(m: dict) -> dict:
    """the motion as the library reads it: every field rounded to float32 first (the C struct), then the axis normalised"""
    n = _f32(m.get("axis", (0.0, 0.0, 1.0)))
    return dict(n=n / np.linalg.norm(n), p=_f32(m.get("pivot", (0.0, 0.0, 0.0))), Th=float(_f32(m.get("roll_amplitude", 0.0))),
                w=float(_f32(m.get("roll_omega", 0.0))), phi=float(_f32(m.get("roll_phase", 0.0))), S=float(_f32(m.get("spin", 0.0))),
                ac=_f32(m.get("accel", (0.0, 0.0, 0.0))),
                harm=[(_f32(h.get("amplitude", (0.0, 0.0, 0.0))), float(_f32(h.get("omega", 0.0))), float(_f32(h.get("phase", 0.0))))
                      for h in m.get("harmonics", ())],
                Tr=float(_f32(m.get("ramp", 0.0))))


def ramp(P, t):
    """(e, e') of the ramp at t"""
    if P["Tr"] > 0.0 and t < P["Tr"]:
        return t / P["Tr"], 1.0 / P["Tr"]
    return 1.0, 0.0


def spin_angle(P, t):
    """theta_s(t) = integral_0^t e(s) Omega0 ds"""
    Tr, S = P["Tr"], P["S"]
    if Tr > 0.0 and t < Tr:
        return S * t * t / (2.0 * Tr)
    return S * (t - Tr / 2.0)


def theta(P, t):
    e, _ = ramp(P, t)
    return e * P["Th"] * np.sin(P["w"] * t + P["phi"]) + spin_angle(P, t)


def rot(n, a):
    """Rot(n, a) as a 3x3 matrix (Rodrigues)"""
    n = np.asarray(n, np.float64)
    K = np.array([[0.0, -n[2], n[1]], [n[2], 0.0, -n[0]], [-n[1], n[0], 0.0]])
    return np.eye(3) + np.sin(a) * K + (1.0 - np.cos(a)) * (K @ K)


def accel(P, t):
    """a_w(t), world"""
    e, _ = ramp(P, t)
    a = P["ac"].copy()
    for A, w, ph in P["harm"]:
        a = a + A * np.sin(w * t + ph)
    return e * a


def state(m: dict, G, t: float) -> np.ndarray:
    """{theta, thd, thdd, R (G - a_w) (3), a_w (3)} at t, float64"""
    P = params(m)
    e, ed = ramp(P, t)
    s, c = np.sin(P["w"] * t + P["phi"]), np.cos(P["w"] * t + P["phi"])
    Th, w, S = P["Th"], P["w"], P["S"]
    thd = ed * Th * s + e * Th * w * c + e * S
    thdd = 2.0 * ed * Th * w * c - e * Th * w * w * s + ed * S
    th = theta(P, t)
    aw = accel(P, t)
    g = rot(P["n"], -th) @ (_f32(G) - aw)
    return np.concatenate([[th, thd, thdd], g, aw])


def step(m: dict, G, t: float, dt: float, x, v):
    """v after one step at t_n = t: Rot(n, -2 thd dt) v + dt (R (G - a_w) - thdd n x r - thd^2 n x (n x r)), r = x - p.
    Returns (v_new, terms) with the float64 terms {coriolis: the rotated v, gravity, euler, centrifugal} per particle."""
    P = params(m)
    st = state(m, G, t)
    thd, thdd, g = st[1], st[2], st[3:6]
    r = np.asarray(x, np.float64) - P["p"]
    nr = np.cross(P["n"], r)
    nnr = np.cross(P["n"], nr)
    vr = np.asarray(v, np.float64) @ rot(P["n"], -2.0 * thd * dt).T
    terms = dict(coriolis=vr, gravity=np.broadcast_to(dt * g, vr.shape), euler=-dt * thdd * nr, centrifugal=-dt * thd * thd * nnr)
    return vr + terms["gravity"] + terms["euler"] + terms["centrifugal"], terms


def accel_bound(m: dict, G, space) -> float:
    """sphk_tank_accel_bound's formula, float64"""
    P = params(m)
    hi = 0.99 * _f32(space)
    far = np.maximum(np.abs(P["p"]), np.abs(hi - P["p"]))
    rmax = float(np.linalg.norm(far))
    Th, w, S = abs(P["Th"]), P["w"], abs(P["S"])
    rinv = 1.0 / P["Tr"] if P["Tr"] > 0.0 else 0.0
    lin = np.linalg.norm(_f32(G)) + np.linalg.norm(P["ac"]) + sum(np.linalg.norm(A) for A, _, _ in P["harm"])
    return float(lin + rmax * (Th * w * w + (2.0 * Th * w + S) * rinv + (Th * w + Th * rinv + S) ** 2))


def sampled_accel(m: dict, G, space, ts) -> float:
    """max over t in ts of |G - a_w| + r_max (|thdd| + thd^2): what accel_bound bounds"""
    P = params(m)
    hi = 0.99 * _f32(space)
    rmax = float(np.linalg.norm(np.maximum(np.abs(P["p"]), np.abs(hi - P["p"]))))
    best = 0.0
    for t in ts:
        st = state(m, G, t)
        best = max(best, np.linalg.norm(_f32(G) - st[6:9]) + rmax * (abs(st[2]) + st[1] ** 2))
    return best
