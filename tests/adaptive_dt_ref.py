"""Reference of CFL-adaptive time stepping (DESIGN.md section 2.8), restated from the documentation in float64 / float32:
the step-size rule of sphk_time_step, the substep partition of SPHSystem::advance and the speed bound of sphk_step_speed."""
import math

import numpy as np

F = np.float32
MIN_CLAMP, NONFINITE, FRAME_END = 1, 2, 4


def rule(C, dt_min, dt_max, R, g, v_max, dt_prev, remaining):
    """(float32 dt, flags) of one step: v_b = v_max + |G| dt_prev, dt = C R / v_b clamped to [dt_min, dt_max], then the frame end."""
    C, dt_min, dt_max, R, g = (float(x) for x in (C, dt_min, dt_max, R, g))
    v_max, dt_prev, remaining = float(v_max), float(dt_prev), float(remaining)
    flags = 0
    if not math.isfinite(v_max):
        dt, flags = dt_min, NONFINITE
    else:
        vb = v_max + g * dt_prev
        dt = C * R / vb if vb > 0 else dt_max
        dt = min(dt, dt_max)
        if dt < dt_min:
            dt, flags = dt_min, MIN_CLAMP
    if remaining > 0:
        if remaining <= dt:
            dt, flags = remaining, flags | FRAME_END
        elif remaining < 2 * dt:
            dt = 0.5 * remaining
    return F(dt), flags


def partition(T, speeds, C, dt_min, dt_max, R, g, dt_prev):
    """the float32 dts advance(T) takes when the k-th substep starts from speed speeds(k); the double sum is accumulated as
    SPHSystem::advance does"""
    elapsed, out = 0.0, []
    while True:
        dt, flags = rule(C, dt_min, dt_max, R, g, speeds(len(out)), dt_prev, T - elapsed)
        out.append(dt)
        elapsed += float(dt)
        dt_prev = float(dt)
        if flags & FRAME_END:
            return out


def fluid_speed(vel):
    """(max |v| over the finite rows, non-finite row count): |v|^2 = (vx vx + vy vy) + vz vz in float32, sqrt in float32"""
    v = np.asarray(vel, F).reshape(-1, 3)
    ok = np.isfinite(v).all(1)
    w = v[ok]
    v2 = (w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1]) + w[:, 2] * w[:, 2]
    return (np.sqrt(v2.max()) if v2.size else F(0)), int((~ok).sum())


def body_speed64(motion, rmax):
    """max over bodies of |V| + |Omega| r_max in float64 (motion: (b, 6) {V, Omega})"""
    m = np.asarray(motion, np.float64).reshape(-1, 6)
    return float((np.linalg.norm(m[:, :3], axis=1) + np.linalg.norm(m[:, 3:], axis=1) * np.asarray(rmax, np.float64)).max())
