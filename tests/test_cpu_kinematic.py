"""The float64 reference of the kinematic bodies (tests/kinematic_ref.py) against closed forms: placement is a rigid
transform, constant-Omega updates compose to one rotation, per-group masses of a lone body are its own ungrouped masses,
and a Galilean motion of fluid and boundary has zero divergence.  Plus the new C-ABI symbols of libsphk.so."""
import os
import subprocess
from types import SimpleNamespace

import numpy as np

import kinematic_ref as KR
import ref64
from util import ROOT

R, SPACING, M0, RHOB = 0.04, 0.02, 76.596750762082e-6, 1.4


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def _pose(seed):
    rng = np.random.default_rng(seed)
    q = _unit(rng.standard_normal(4))
    return np.concatenate([rng.uniform(0.2, 0.8, 3), q]), np.concatenate([rng.uniform(-1, 1, 3), rng.uniform(-5, 5, 3)])


def _slab(nx=8, ny=6):
    i, j, k = np.meshgrid(np.arange(nx), np.arange(ny), np.arange(2), indexing="ij")
    return np.stack([(i - 0.5 * (nx - 1)) * SPACING, (j - 0.5 * (ny - 1)) * SPACING, (k - 0.5) * SPACING], -1).reshape(-1, 3)


def test_placement_is_a_rigid_transform():
    r = _slab() + np.random.default_rng(4).uniform(-0.003, 0.003, (96, 3))
    for seed in range(5):
        pose, motion = _pose(seed)
        x, v = KR.place(pose, motion, r)
        d0 = np.linalg.norm(r[:, None] - r[None], axis=-1)
        d1 = np.linalg.norm(x[:, None] - x[None], axis=-1)
        assert np.abs(d1 - d0).max() <= 1e-12
        Rm = KR.rotation(pose[3:])
        assert np.abs(Rm @ Rm.T - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(Rm) - 1.0) <= 1e-12
        # rigid velocity field: (v_i - v_j) . (x_i - x_j) = 0
        assert np.abs(((v[:, None] - v[None]) * (x[:, None] - x[None])).sum(-1)).max() <= 1e-12
        assert np.allclose(v, motion[:3] + np.cross(motion[3:], x - pose[:3]), atol=1e-12)


def test_constant_omega_updates_compose_to_one_rotation():
    for seed in range(4):
        pose, motion = _pose(seed + 10)
        dt, N = 0.004, 250
        p = pose.copy()
        for _ in range(N):
            p = KR.pose_update(p, motion, dt)
        W = motion[3:]
        w = np.linalg.norm(W)
        ang = w * N * dt
        q_exact = KR.quat_mul(np.concatenate([np.sin(ang / 2) * W / w, [np.cos(ang / 2)]]), pose[3:])
        assert np.abs(p[3:] - q_exact).max() <= 1e-12
        assert np.abs(p[:3] - (pose[:3] + N * dt * motion[:3])).max() <= 1e-12
    # Omega = 0: the orientation does not change at all
    pose, motion = _pose(99)
    motion[3:] = 0.0
    assert np.array_equal(KR.pose_update(pose, motion, 0.004)[3:], pose[3:])


def test_lone_body_grouped_masses_equal_its_own_ungrouped_masses():
    r = _slab()
    pose, _ = _pose(3)
    x, _ = KR.place(pose, np.zeros(6), r)
    # a static set far away from the body: the grouping changes nothing for either
    wall = np.stack(np.meshgrid(np.arange(10) * SPACING, [0.0], np.arange(10) * SPACING, indexing="ij"), -1).reshape(-1, 3) + [3.0, 0, 0]
    allp = np.concatenate([wall, x])
    group = np.concatenate([np.zeros(len(wall), int), np.ones(len(x), int)])
    m = KR.grouped_masses(allp, group, RHOB, R)
    alone = KR.grouped_masses(x, np.zeros(len(x), int), RHOB, R)
    assert np.abs(m[len(wall):] - alone).max() <= 1e-12 * alone.max()
    # and two touching groups do not see each other: a copy of the body moved by R / 2 keeps the same masses
    both = np.concatenate([x, x + [R / 2, 0, 0]])
    mg = KR.grouped_masses(both, np.repeat([1, 2], len(x)), RHOB, R)
    assert np.abs(mg[:len(x)] - alone).max() <= 1e-12 * alone.max() and np.abs(mg[len(x):] - alone).max() <= 1e-12 * alone.max()


def test_galilean_motion_has_zero_divergence():
    g = np.arange(8) * SPACING + 0.1
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    pos = pos + np.random.default_rng(1).uniform(-0.003, 0.003, pos.shape)
    posB = KR.place(np.array([0.17, 0.17 - 0.0, 0.17, 0, 0, 0, 1.0]), np.zeros(6), _slab(6, 6))[0]
    pos = pos[np.min(np.linalg.norm(pos[:, None] - posB[None], axis=-1), 1) > SPACING]
    A = SimpleNamespace(posF=pos, massF=np.full(len(pos), M0), csF=np.array([0, len(pos)]), posB=posB,
                        massB=np.full(len(posB), 2 * M0), csB=np.array([0, len(posB)]), g=SimpleNamespace(ncells=1), R=R)
    P = ref64.Pairs(A)
    assert len(P.iB) > 0
    V = np.array([0.3, -0.2, 0.7])
    s, m = KR.divergence(P, np.tile(V, (len(pos), 1)), np.tile(V, (len(posB), 1)))
    assert np.all(s == 0.0) and np.all(m == 0.0)
    # a boundary at rest against moving fluid does not vanish (the term the bodies add)
    s1, _ = KR.divergence(P, np.tile(V, (len(pos), 1)), np.zeros((len(posB), 3)))
    assert np.abs(s1).max() > 0
    # and with v_b = 0 it is ref64's divergence
    e0, _ = ref64._divergence(P, np.tile(V, (len(pos), 1)))
    assert np.array_equal(s1, e0)


def test_body_symbols_are_exported(built):
    lib = os.path.join(ROOT, "cpp-fluid-particles_b200", "libsphk.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], stdout=subprocess.PIPE, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if " T " in line}
    for f in ("sphk_bodies_init", "sphk_bodies_set_motion", "sphk_bodies_step", "sphk_bodies_get_pose", "sphk_bodies_get_local"):
        assert f in names, f
    host = os.path.join(ROOT, "cpp-fluid-particles_b200", "libsphhost.so")
    out = subprocess.run(["nm", "-D", "--defined-only", host], stdout=subprocess.PIPE, text=True, check=True).stdout
    for f in ("sph_app_create_with_bodies", "sph_app_set_body_motion", "sph_app_body_pose"):
        assert f in out, f
