"""The float64 reference of two-way coupled bodies (tests/rigid_ref.py) against closed forms, and the exported names."""
import os
import subprocess

import numpy as np

import rigid_ref as RR
from util import ROOT
from kinematic_ref import rotation

RNG = np.random.default_rng(11)


def _unit(q):
    q = np.asarray(q, np.float64)
    return q / np.linalg.norm(q)


def test_torque_free_body_keeps_its_angular_momentum():
    """H = 0: L = Iw(q) Omega is unchanged by the update, at any orientation"""
    q = _unit(RNG.standard_normal(4))
    I = np.array([0.3, 1.1, 2.7])
    m0 = np.array([0.1, -0.2, 0.05, 1.3, -0.4, 2.2])
    m1 = RR.integrate(m0, q, 2.0, I, np.zeros(3), np.zeros(3), 0.004, np.zeros(3))
    Iw = RR.world_inertia(q, I)
    assert np.allclose(Iw @ m1[3:], Iw @ m0[3:], rtol=0, atol=1e-12)
    assert np.array_equal(m1[:3], m0[:3])


def test_spherical_body_keeps_its_angular_velocity():
    q = _unit(RNG.standard_normal(4))
    m0 = np.array([0.0, 0.0, 0.0, 0.7, -1.9, 0.3])
    m1 = RR.integrate(m0, q, 5.0, [0.8, 0.8, 0.8], np.zeros(3), np.zeros(3), 0.004, np.zeros(3))
    assert np.allclose(m1[3:], m0[3:], rtol=0, atol=1e-12)


def test_integrator_matches_closed_forms_for_constant_impulses():
    """N steps of constant J and H: V = V0 + N (J/M + dt G); at a fixed orientation Omega = Omega0 + N Iw^-1 H"""
    q = _unit(RNG.standard_normal(4))
    I, M, dt, G = np.array([0.5, 1.5, 2.5]), 3.0, 0.004, np.array([0.0, -9.8, 0.0])
    J, H = np.array([0.01, 0.03, -0.02]), np.array([-0.002, 0.004, 0.001])
    m = np.array([0.1, 0.0, -0.1, 0.2, 0.0, 0.4])
    N = 25
    m0 = m.copy()
    for _ in range(N):
        m = RR.integrate(m, q, M, I, J, H, dt, G)
    assert np.allclose(m[:3], m0[:3] + N * (J / M + dt * G), rtol=0, atol=1e-12)
    assert np.allclose(m[3:], m0[3:] + N * np.linalg.solve(RR.world_inertia(q, I), H), rtol=0, atol=1e-12)
    # about a principal axis at the identity orientation: dOmega_a = H_a / I_a
    m1 = RR.integrate(np.zeros(6), [0, 0, 0, 1], M, I, np.zeros(3), H, dt, np.zeros(3))
    assert np.allclose(m1[3:], H / I, rtol=0, atol=1e-15)


def test_contact_puts_the_box_back_and_zeroes_only_the_outward_velocity():
    lo, hi, clamp = np.array([-0.05, -0.04, -0.03]), np.array([0.05, 0.04, 0.03]), np.array([0.99, 0.99, 0.99])
    q = _unit([0.1, 0.3, -0.2, 0.9])
    # through the floor and the +x wall, moving outward on both, inward on z
    c, V = RR.contact([0.97, 0.01, 0.5], q, [0.3, -0.5, 0.2], lo, hi, clamp)
    corners = np.array([[(hi if s & 1 else lo)[0], (hi if s & 2 else lo)[1], (hi if s & 4 else lo)[2]] for s in range(8)])
    x = c + corners @ rotation(q).T
    assert x.min() >= -1e-12 and (x.max(0) <= clamp + 1e-12).all()
    assert abs(x[:, 1].min()) < 1e-12 and abs(x[:, 0].max() - clamp[0]) < 1e-12, "touching, not pushed further"
    assert V[0] == 0.0 and V[1] == 0.0 and V[2] == 0.2
    # moving inward already: the velocity is kept, the position still corrected
    c2, V2 = RR.contact([0.5, 0.01, 0.5], q, [0.0, 0.5, 0.0], lo, hi, clamp)
    assert np.array_equal(V2, [0.0, 0.5, 0.0]) and c2[1] > 0.01
    # inside: nothing changes
    c3, V3 = RR.contact([0.5, 0.5, 0.5], q, [1.0, -1.0, 1.0], lo, hi, clamp)
    assert np.array_equal(c3, [0.5, 0.5, 0.5]) and np.array_equal(V3, [1.0, -1.0, 1.0])


def test_symmetric_body_in_a_uniform_lattice_feels_no_net_force():
    """a cube of body particles centred in a uniform fluid lattice with uniform s: the reaction sums to zero force and
    torque (every pair term has its mirror image)"""
    h = 0.02
    R = 2 * h
    ax = (np.arange(-8, 9)) * h
    xf = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3) + 0.5
    bx = (np.arange(-2, 3)) * h
    cube = np.stack(np.meshgrid(bx, bx, bx, indexing="ij"), -1).reshape(-1, 3)
    cube = cube[(np.abs(cube) > 1.5 * h).any(1)] + 0.5 + 0.5 * h        # hollow, centred between lattice points
    n = len(xf)
    JH, mag = RR.reaction(xf, np.full(n, 0.37), np.full(n, 7.6e-5), cube, np.full(len(cube), 5e-5),
                          np.zeros(len(cube), int), [np.full(3, 0.5 + 0.5 * h)], 1.0, R)
    assert (mag[0] > 0).all()
    assert (np.abs(JH[0]) <= 1e-12 * mag[0]).all(), (JH, mag)
    # the same body off-centre in the lattice's top layer feels a net force (the test can fail)
    JH2, _ = RR.reaction(xf, np.full(n, 0.37), np.full(n, 7.6e-5), cube + [0, 7 * h, 0], np.full(len(cube), 5e-5),
                         np.zeros(len(cube), int), [np.full(3, 0.5 + 7.5 * h)], 1.0, R)
    assert abs(JH2[0, 1]) > 1e-3 * np.abs(mag[0]).max()


def test_new_entries_are_exported(pkg, built):
    capi = pkg.capi
    for name in ("sphk_bodies_set_dynamics", "sphk_bodies_react", "sphk_bodies_integrate", "sphk_bodies_set_body_motion",
                 "sphk_bodies_get_motion", "sphk_bodies_get_impulse"):
        assert name in capi.SPHK_FUNCTIONS
    for name in ("sph_app_create_with_dynamic_bodies", "sph_app_body_motion", "sph_app_body_impulse"):
        assert name in capi.SPH_APP_FUNCTIONS
    for lib, names in (("libsphk.so", capi.SPHK_FUNCTIONS[-6:]), ("libsphhost.so", capi.SPH_APP_FUNCTIONS[-3:])):
        out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "cpp-fluid-particles_b200", lib)],
                             stdout=subprocess.PIPE, text=True, check=True).stdout
        for f in names:
            assert f in out, f
    mi = capi.body_mass_inertia([{"mass": 2.0, "inertia": (1, 2, 3)}, {}])
    assert mi.dtype == np.float32 and mi.tolist() == [[2, 1, 2, 3], [0, 0, 0, 0]]
