"""CPU checks of the oracle on the reference's default 40-object scene (UR5gripper_2_finger_many_objects.xml): the closed-form
narrow-phase pairs added for capsules / cylinders against hand-computed configurations, the reset rule of GraspingEnv.py:418-430,
and a settle run (objects end up resting on the table or the floor, contacts condim 6, deterministic)."""
import numpy as np
import pytest

from tests.common import HOME, contact_is_analytic, reset_qpos_scene_b

S2 = np.sqrt(0.5)


@pytest.fixture(scope="module")
def orcb(scene_b):
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(scene_b[0])
    yield o
    o.close()


def _parked(A):
    """all 40 objects far apart and far above everything (no contacts), arm at HOME"""
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(40):
        a = 8 + 7 * i
        q[a:a + 7] = [3.0 + i, 5.0, 6.0, 1, 0, 0, 0]
    return q


def _place(q, i, pos, quat=(1, 0, 0, 0)):
    a = 8 + 7 * i
    q[a:a + 3] = pos
    q[a + 3:a + 7] = quat


def _contacts_between(o, g1, g2):
    c = o.contacts()
    return c[(c[:, 13] == g1) & (c[:, 14] == g2)]


def test_closed_form_pairs_for_capsules_and_cylinders(orcb, scene_b):
    _, A, _ = scene_b
    size = np.asarray(A["geom_size"]).reshape(-1, 3)
    gtype = np.asarray(A["geom_type"])
    sph, box, cyl, cap = 30, 40, 50, 60  # first geom of each object family (object i = geom 30 + i)
    assert gtype[sph] == 2 and gtype[box] == 6 and gtype[cyl] == 5 and gtype[cap] == 3
    q = _parked(A)
    # sphere 0 beside capsule 30 (axis z): closest axis point at the sphere's height
    rs, rc = size[sph, 0], size[cap, 0]
    _place(q, 30, [0, 0, 3.0]); _place(q, 0, [rs + rc - 0.002, 0, 3.01])
    # sphere 1 on top of cylinder 20 (axis z)
    rs1, hc = size[sph + 1, 0], size[cyl, 1]
    _place(q, 20, [2, 0, 3.0]); _place(q, 1, [2.003, 0.001, 3.0 + hc + rs1 - 0.001])
    # capsule 31 (axis z) crossed with capsule 32 turned about x (axis -> y)
    r1, r2 = size[cap + 1, 0], size[cap + 2, 0]
    _place(q, 31, [4, 0, 3.0]); _place(q, 32, [4 + r1 + r2 - 0.003, 0, 3.0], [S2, S2, 0, 0])
    # capsule 33 lying on the floor plane (axis -> x), cylinder 21 standing on the floor
    r3, h3 = size[cap + 3, 0], size[cap + 3, 1]
    _place(q, 33, [6, 3, r3 - 0.001], [S2, 0, S2, 0])
    h21 = size[cyl + 1, 1]
    _place(q, 21, [8, 3, h21 - 0.0005])
    orcb.reset(q)
    orcb.forward()
    c = _contacts_between(orcb, sph, cap)
    assert len(c) == 1 and abs(c[0, 0] + 0.002) < 1e-12 and np.allclose(c[0, 4:7], [-1, 0, 0], atol=1e-12)
    assert np.allclose(c[0, 1:4], [rs + rc - 0.002 - (rs - 0.001), 0, 3.01], atol=1e-12)
    c = _contacts_between(orcb, sph + 1, cyl)
    assert len(c) == 1 and abs(c[0, 0] + 0.001) < 1e-12 and np.allclose(c[0, 4:7], [0, 0, -1], atol=1e-12)
    c = _contacts_between(orcb, cap + 1, cap + 2)
    assert len(c) == 1 and abs(c[0, 0] + 0.003) < 1e-9 and np.allclose(c[0, 4:7], [1, 0, 0], atol=1e-9)
    assert np.allclose(c[0, 1:4], [4 + r1 - 0.0015, 0, 3.0], atol=1e-9)
    c = _contacts_between(orcb, 0, cap + 3)  # geom 0 = the floor plane
    assert len(c) == 2 and np.allclose(c[:, 0], -0.001, atol=1e-9) and np.allclose(c[:, 4:7], [[0, 0, 1]] * 2, atol=1e-12)
    assert np.allclose(sorted(c[:, 1]), [6 - h3, 6 + h3], atol=1e-9)
    c = _contacts_between(orcb, 0, cyl + 1)
    assert len(c) == 1 and abs(c[0, 0] + 0.0005) < 1e-9 and np.allclose(c[0, 1:3], [8, 3], atol=1e-9)
    assert (orcb.contacts()[:, 15] == 6).all()  # condim 6 everywhere in this scene
    assert orcb.ncon == 6


def test_reset_rule_matches_the_reference_draw_order(scene_b):
    from mujoco_rl_ur5_b200.batched_env import random_unit_quaternion, scene_b_reset_qpos

    _, A, _ = scene_b
    for i in (0, 7):
        q = scene_b_reset_qpos(A, 20000 + i)
        assert np.array_equal(q, reset_qpos_scene_b(A, i))
        obj = q[8:].reshape(40, 7)
        assert (np.abs(obj[:, 0]) <= 0.25).all() and (obj[:, 1] >= -0.77).all() and (obj[:, 1] <= -0.43).all()
        assert (obj[:, 2] >= 1.0).all() and (obj[:, 2] <= 1.5).all()
        assert np.allclose(np.linalg.norm(obj[:, 3:], axis=1), 1.0, atol=1e-12)
    # pyquaternion's Quaternion.random(): (sqrt(1-r1) sin 2 pi r2, sqrt(1-r1) cos 2 pi r2, sqrt(r1) sin 2 pi r3, sqrt(r1) cos 2 pi r3)
    assert np.allclose(random_unit_quaternion(0.25, 0.25, 0.5), [np.sqrt(0.75), 0, 0, -0.5], atol=1e-12)
    # numpy's global stream, like the reference
    np.random.seed(11)
    a = scene_b_reset_qpos(A)
    np.random.seed(11)
    assert np.array_equal(a, scene_b_reset_qpos(A))


def test_objects_fall_and_come_to_rest(orcb, scene_b):
    _, A, _ = scene_b
    q0 = reset_qpos_scene_b(A, 3)
    orcb.reset(q0)
    orcb.move_group("All", HOME + 0.05, 1e-9, 599)
    q1 = orcb.qpos.copy()
    z = q1[10:288:7]
    assert orcb.ncon >= 25 and (orcb.contacts()[:, 15] == 6).all()
    assert ((z > 0.88) & (z < 1.1) | (z > 0.0) & (z < 0.1)).all(), z  # on the table (0.9 + half size) or on the floor beside it
    assert ((z > 0.88) & (z < 1.1)).sum() >= 30
    assert np.isfinite(orcb.qvel).all() and np.abs(orcb.qvel[8:]).max() < 6.0
    orcb.reset(q0)
    orcb.move_group("All", HOME + 0.05, 1e-9, 599)
    assert np.array_equal(q1, orcb.qpos)  # deterministic


def test_contact_capacity_keeps_a_prefix_of_the_emission_order(scene_b):
    """set_maxcon(n): the list is the first n contacts of the uncapped list (analytic pairs, then MPR pairs), the overflow flag is
    set iff the uncapped count exceeds n, and the default capacity gives the same results as before any cap was set"""
    from oracle.oracle_py import OracleEnv

    blob, A, _ = scene_b
    o = OracleEnv(blob)
    o.reset(reset_qpos_scene_b(A, 3))
    o.move_group("All", HOME + 0.05, 1e-9, 399)
    q, v = o.qpos.copy(), o.qvel.copy()
    o.reset(q, v)
    o.forward()
    full, total = o.contacts(), o.ncon
    acc, frc = o.field("qacc"), o.field("qfrc_constraint")
    assert total >= 25 and o.con_overflow == 0
    analytic = contact_is_analytic(A, full)
    n_analytic = int(analytic.sum())
    assert 0 < n_analytic < total and analytic[:n_analytic].all()  # analytic contacts first, then the MPR ones
    for cap in (total + 5, total, total - 1, n_analytic + (total - n_analytic) // 2, n_analytic, 16, 0):
        o.set_maxcon(cap)
        o.reset(q, v)
        o.forward()
        assert o.ncon == min(cap, total), cap
        assert np.array_equal(o.contacts(), full[:min(cap, total)]), cap
        assert o.con_overflow == int(total > cap), cap
        assert np.isfinite(o.field("qacc")).all()
    o.set_maxcon(256)
    o.reset(q, v)
    o.forward()
    assert o.ncon == total and o.con_overflow == 0
    assert np.array_equal(o.field("qacc"), acc) and np.array_equal(o.field("qfrc_constraint"), frc)
    o.close()
