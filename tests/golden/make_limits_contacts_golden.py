#!/usr/bin/env python
"""Generates tests/golden/limits_contacts.npz: constructed states that take the solver's joint-limit rows, the 16 simple-row slots and
the degenerate branches of the narrow phase (tests/test_limits_contacts_gpu.py).

TEST INFRASTRUCTURE.  No stored fixture state before this one builds a joint-limit row (efc_type 1) or reaches the closed-form
branches where a contact function divides by something near zero or picks between ties; tools/oracle_branch_coverage.py measures this.
Every state here is built by hand and tagged with the branch it targets:
  * scene A, limits: one limit per state (shoulder_lift past 0, wrist_1 past -pi, wrist_3 past +pi, both fingers past +-1 through the
    finger equality, an object slide past +-5 in x or y or past +2 in z with the object out of contact), each at the depths 0.0002,
    0.0007 and 0.003, which put `impedance` (width 0.001, mid 0.5) in its x <= mid, mid < x < 1 and x >= 1 branch; the joint moves into
    the limit in some states and away from it in others, so that both active and inactive limit rows occur;
  * scene A, capacity: 14, 15 and 16 limit rows besides the equality row (15 and 16 simple rows fit GE_MAXSR = 16, 17 overflow);
  * scene A, trajectories: the start of an open-loop run that drives shoulder_lift into its upper limit, pulls it back and pushes it
    in again, and the start of a move_group whose target lies beyond that limit (the tests replay both; the commands are stored here);
  * scene B (CTA-per-env build, objects parked apart in the air): arm and finger limits, one state with five limits at once;
  * degenerate contacts, scene A: a ball's centre inside a box (each box axis once as the axis of least depth, both signs), two balls
    with coincident centres, an axis-aligned box-on-box stack (face-axis ties of the SAT, decided by a strict `>`);
  * degenerate contacts, scene B: parallel capsules side by side, crossing capsules whose axes intersect, a sphere centre inside a
    cylinder (radial and axial distance deciding), a sphere centre on a capsule axis, an exactly upright cylinder on the floor, and a
    capsule standing coaxially on an upright cylinder (an MPR pair: the cylinder's support along its axis, the origin on the
    centre -> v1 ray).
col_plane_mesh: no arm pose inside the joint ranges brings an arm mesh within reach of the floor (the shoulder sits at z 0.96 on top
of its stand and shoulder_lift keeps the upper arm above the horizontal), so no state of this file calls it.
A state is kept only if the oracle's -ffp-contract=fast build takes the same branches (same contacts, rows, row split and Newton
iterations) and agrees with the checker build within a tenth of the GPU tests' tolerances: analytic contacts 1e-10, MPR contacts 1e-8,
qacc and qfrc_constraint 1e-8 relative.

The .npz is written with fixed zip timestamps, so a rerun reproduces the committed file byte for byte.

  python tests/golden/make_limits_contacts_golden.py      (a few seconds)
"""
import io
import os
import subprocess
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "limits_contacts.npz")
HOME = np.array([0, -1.57, 1.57, -1.57, -1.57, 0.0, 0.3])
DEPTHS = (0.0002, 0.0007, 0.003)  # impedance x = depth / width: 0.2 (<= mid), 0.7 (mid < x < 1), 3 (>= 1)
PEN = 5e-4
FIRST_OBJ_BODY_A = 18
Q_HALF = np.sqrt(0.5)
QUAT_X = np.array([Q_HALF, 0, Q_HALF, 0])  # local z along world x
QUAT_Y = np.array([Q_HALF, -Q_HALF, 0, 0])  # local z along world y
# with the elbow at -0.5 the arm touches nothing while shoulder_lift is near its upper limit (at HOME's 1.57 the forearm lies on the
# drop bin, and the MPR contacts of its meshes make the trajectory diverge between the oracle's two builds within 10 sub-steps)
ELBOW_CLEAR = -0.5
# the open-loop run, shoulder_lift 0.02 below its upper limit: pushed up (its limit row turns active), pulled back for 3 sub-steps (the
# row stays, inactive) and pushed up again (active); the move_group target lies past that limit
OPEN_LOOP_CTRL = np.array([[0.0, 1.0, 0, 0, 0, 0, 0], [0.0, -2.0, 0, 0, 0, 0, 0], [0.0, 1.0, 0, 0, 0, 0, 0]])
OPEN_LOOP_STEPS = np.array([40, 3, 40], np.int32)
BEYOND_TARGET = np.array([0.0, 0.25, ELBOW_CLEAR, -1.57, -1.57, 0.0, 0.3])
BEYOND_STEPS = 80


def _scenes():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    return {s: (load_scene_blob(s), load_scene(s)[0]) for s in "AB"}


def _base_a(A):
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(6):
        _place_a(A, q, i, [2.0 + 0.3 * i, 2.0, 1.5])
    return q


def _place_a(A, q, i, world):
    """scene-A object i (0-2 box_1-3, 3-5 ball_1-3): its x / y / z slides are measured from the body's position"""
    bp = np.asarray(A["body_pos"]).reshape(-1, 3)[FIRST_OBJ_BODY_A + i]
    q[8 + 7 * i:11 + 7 * i] = np.asarray(world) - bp
    q[11 + 7 * i:15 + 7 * i] = (1, 0, 0, 0)


def _base_b(A):
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(40):  # free joints: qpos is the world position; a 5 x 8 grid in the air, 0.3 m apart
        _place_b(q, i, [2.0 + 0.3 * (i % 5), 2.0 + 0.3 * (i // 5), 3.0])
    return q


def _place_b(q, i, world, quat=(1, 0, 0, 0)):
    q[8 + 7 * i:11 + 7 * i] = world
    q[11 + 7 * i:15 + 7 * i] = quat


def limit_states_a(A):
    """(tag, qpos, qvel): one limit per state at the three depths; the sign of the velocity alternates (into / away from the limit)"""
    out = []
    rng = np.asarray(A["jnt_range"]).reshape(-1, 2)
    nv = int(np.asarray(A["nv"]).ravel()[0])
    for k, d in enumerate(DEPTHS):
        into = 1.0 if k != 1 else -1.0  # the middle depth moves away from the limit, fast enough to leave the row inactive
        # shoulder_lift up, wrist_1 down, wrist_3 up, fingers up (fingers past -1 press into each other: their mesh contacts are
        # rounding-sensitive between the oracle's two builds)
        for j, side in ((1, 1), (3, 0), (5, 1), (6, 1)):
            q, v = _base_a(A), np.zeros(nv)
            lim = rng[j, side]
            sgn = 1.0 if side else -1.0
            q[j] = lim + sgn * d
            v[j] = sgn * into * (0.05 if into > 0 else 0.6)
            if j == 1:
                q[2] = ELBOW_CLEAR
            if j == 6:  # the finger equality q7 = q6 holds; base_to_rik is past the same limit
                q[7], v[7] = q[6], v[6]
            out.append(("limit j%d %s d%g %s" % (j, "upper" if side else "lower", d, "into" if into > 0 else "away"), q, v))
        for obj, axis, side in ((0, 0, 1), (3, 1, 0), (4, 2, 1)):  # box_1 x past +5, ball_1 y past -5, ball_2 z past +2
            q, v = _base_a(A), np.zeros(nv)
            j = 8 + 4 * obj + axis
            a = 8 + 7 * obj + axis
            lim = rng[j, side]
            sgn = 1.0 if side else -1.0
            q[a] = lim + sgn * d
            v[8 + 6 * obj + axis] = sgn * into * (0.05 if into > 0 else 0.6)
            out.append(("limit slide obj%d axis%d %s d%g" % (obj, axis, "upper" if side else "lower", d), q, v))
    return out


def capacity_states_a(A):
    """14, 15 and 16 limit rows besides the equality row: five arm rows (shoulder_lift, wrist_1, wrist_3, both fingers), then object
    slides in joint order, x past +-5 and z past +2 per object; each object at its own y, so that none touches another"""
    out = []
    rng = np.asarray(A["jnt_range"]).reshape(-1, 2)
    nv = int(np.asarray(A["nv"]).ravel()[0])
    bp = np.asarray(A["body_pos"]).reshape(-1, 3)
    for nlim in (14, 15, 16):
        q, v = _base_a(A), np.zeros(nv)
        q[1], v[1] = 0.0007, 0.02  # shoulder_lift past its upper limit, moving in
        q[3], v[3] = rng[3, 0] - 0.003, 0.3  # wrist_1 past -pi, moving out
        q[2] = rng[2, 1]  # elbow exactly at its upper limit: distance 0 is not below the margin, no row
        q[5] = rng[5, 1] + 0.0002
        q[6] = q[7] = 1.0 + 0.0007  # both fingers past +1
        rows = 5
        for obj in range(6):
            w = np.array([2.0, 0.3 * obj - 1.0, 1.5])
            for axis in (0, 2):
                if rows < nlim:
                    d = DEPTHS[(obj + axis) % 3]
                    sx = 1.0 if obj % 2 == 0 or axis == 2 else -1.0
                    w[axis] = bp[FIRST_OBJ_BODY_A + obj, axis] + sx * (5.0 if axis == 0 else 2.0) + sx * d
                    v[8 + 6 * obj + axis] = 0.04 * (1 if obj % 2 else -1)
                    rows += 1
            _place_a(A, q, obj, w)
        out.append(("capacity %d limit rows" % nlim, q, v))
    return out


def trajectory_states_a(A):
    nv = int(np.asarray(A["nv"]).ravel()[0])
    q, v = _base_a(A), np.zeros(nv)
    q[1], q[2] = -0.02, ELBOW_CLEAR
    q2, v2 = _base_a(A), np.zeros(nv)
    q2[1], q2[2] = -0.15, ELBOW_CLEAR
    return [("open loop into shoulder_lift's upper limit", q, v), ("move_group beyond shoulder_lift's upper limit", q2, v2)]


def contact_states_a(A):
    out = []
    nv = int(np.asarray(A["nv"]).ravel()[0])
    c = np.array([0.0, 1.0, 1.5])  # in the air, out of reach of the arm and the tables
    for k, off in enumerate(([0.01, 0, 0], [0, -0.012, 0.003], [0.002, 0.004, 0.011])):  # x, y (negative side), z least deep
        q = _base_a(A)
        _place_a(A, q, 2, c)  # box_3 (half 0.025)
        _place_a(A, q, 3, c + np.array(off))  # ball_1 (r 0.03) centred inside it
        out.append(("sphere centre inside box axis%d" % k, q, np.zeros(nv)))
    q = _base_a(A)
    _place_a(A, q, 3, c)
    _place_a(A, q, 4, c)  # ball_1 and ball_2 share their centre
    out.append(("sphere-sphere coincident centres", q, np.zeros(nv)))
    q = _base_a(A)
    _place_a(A, q, 2, c)  # box_3 below, box_1 (half 0.02) on its top face, both axis-aligned: the face axes of both boxes tie
    _place_a(A, q, 0, c + np.array([0.003, -0.002, 0.025 + 0.02 - PEN]))
    out.append(("aligned box-box stack", q, np.zeros(nv)))
    return out


def limit_states_b(A):
    out = []
    rng = np.asarray(A["jnt_range"]).reshape(-1, 2)
    nv = int(np.asarray(A["nv"]).ravel()[0])
    for k, d in enumerate(DEPTHS):
        for j, side in ((1, 1), (4, 0), (6, 1)):
            q, v = _base_b(A), np.zeros(nv)
            sgn = 1.0 if side else -1.0
            q[j] = rng[j, side] + sgn * d
            v[j] = sgn * (0.05 if k != 1 else -0.6)
            if j == 1:
                q[2] = ELBOW_CLEAR
            if j == 6:
                q[7], v[7] = q[6], v[6]
            out.append(("B limit j%d %s d%g" % (j, "upper" if side else "lower", d), q, v))
    q, v = _base_b(A), np.zeros(nv)
    q[1], v[1] = 0.0007, 0.05
    q[2], v[2] = rng[2, 1] + 0.003, -0.6
    q[5], v[5] = rng[5, 0] - 0.0002, 0.0
    q[6] = q[7] = 1.0 + 0.0007
    out.append(("B five limits at once", q, v))
    return out


def contact_states_b(A):
    out = []
    nv = int(np.asarray(A["nv"]).ravel()[0])
    c = np.array([-1.0, 1.0, 2.0])  # in the air
    q = _base_b(A)  # capsules object_30 (r .025, h .05) and object_31 (r .025, h .04), both along x, side by side, offset along x
    _place_b(q, 30, c, QUAT_X)
    _place_b(q, 31, c + np.array([0.03, 0.05 - PEN, 0.0]), QUAT_X)
    out.append(("capsule-capsule parallel", q, np.zeros(nv)))
    q = _base_b(A)  # object_30 along x, object_32 (r .015, h .05) along y: the axes cross at x = 0.02 from object_30's centre
    _place_b(q, 30, c, QUAT_X)
    _place_b(q, 32, c + np.array([0.02, 0.0, 0.0]), QUAT_Y)
    out.append(("capsule-capsule crossing axes", q, np.zeros(nv)))
    for tag, off in (("radial", [0.02, 0.0, 0.01]), ("axial", [0.003, 0.004, -0.045])):  # cylinder object_20 (r .025, h .05)
        q = _base_b(A)
        _place_b(q, 20, c)
        _place_b(q, 0, c + np.array(off))  # sphere object_0 (r .03)
        out.append(("sphere centre inside cylinder, %s" % tag, q, np.zeros(nv)))
    q = _base_b(A)
    _place_b(q, 30, c, QUAT_X)
    _place_b(q, 1, c + np.array([-0.02, 0.0, 0.0]))  # sphere object_1 on object_30's axis
    out.append(("sphere centre on capsule axis", q, np.zeros(nv)))
    q = _base_b(A)
    _place_b(q, 21, [-1.0, 1.5, 0.04 - PEN])  # cylinder object_21 (r .025, h .04) upright on the floor
    out.append(("upright cylinder on the floor", q, np.zeros(nv)))
    q = _base_b(A)
    _place_b(q, 20, [-1.0, 1.5, 0.05 - PEN])  # cylinder object_20 upright on the floor, capsule object_33 (r .02, h .05) on top of it
    _place_b(q, 33, [-1.0, 1.5, 0.1 - 2 * PEN + 0.05 + 0.02 - PEN])
    out.append(("capsule coaxial on upright cylinder", q, np.zeros(nv)))
    return out


def measure(args):
    """per state: contacts, the row split, qacc (and the capped row split / qacc for the capacity states)"""
    items, so = args
    if so:
        os.environ["GRASP_ORACLE_SO"] = so
    from oracle.oracle_py import OracleEnv

    sc = _scenes()
    res = []
    for scene, tag, q, v in items:
        o = OracleEnv(sc[scene][0])
        o.reset(q, v)
        o.forward()
        res.append((o.contacts(), (o.efc_split, o.solver_iter), o.field("qacc"), o.field("qfrc_constraint")))
        o.close()
    return res


def robust(a, b, A):
    """the checker and the fast build take the same branches (contacts, rows, Newton iterations) and agree within a tenth of the
    GPU tests' bars"""
    from tests.common import contact_is_analytic

    (ca, sa, qa, fa), (cb, sb, qb, fb) = a, b
    if sa != sb or ca.shape != cb.shape or not np.array_equal(ca[:, 13:], cb[:, 13:]):
        return False
    if len(ca):
        tol = np.where(contact_is_analytic(A, ca), 1e-10, 1e-8)
        if (np.abs(ca[:, :13] - cb[:, :13]).max(axis=1) >= tol).any():
            return False
    return all(np.abs(x - y).max() <= 1e-8 * max(1.0, float(np.abs(x).max())) for x, y in ((qa, qb), (fa, fb)))


def save_npz(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member (np.savez stamps the current time)"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "fast"])
    fast = os.path.join(ROOT, "oracle", "libgrasp_oracle_fast.so")
    sc = _scenes()
    A, B = sc["A"][1], sc["B"][1]
    items = [("A",) + s for s in limit_states_a(A) + capacity_states_a(A) + trajectory_states_a(A) + contact_states_a(A)]
    items += [("B",) + s for s in limit_states_b(B) + contact_states_b(B)]
    from multiprocessing import Pool

    with Pool(2, maxtasksperchild=1) as pool:
        ref, alt = pool.map(measure, [(items, None), (items, fast)])
    kept = {"A": [], "B": []}
    for it, a, b in zip(items, ref, alt):
        ok = robust(a, b, sc[it[0]][1])
        print("%s %-48s rows (eq, limit, contact), Newton iterations %-18s ncon %2d %s" % (it[0], it[1], a[1], len(a[0]),
                                                                                         "" if ok else "DROPPED: rounding-sensitive"))
        if ok:
            kept[it[0]].append(it)
    arrays = {}
    for s, sfx in (("A", "_a"), ("B", "_b")):
        arrays["qpos" + sfx] = np.array([it[2] for it in kept[s]])
        arrays["qvel" + sfx] = np.array([it[3] for it in kept[s]])
        arrays["tag" + sfx] = np.array([it[1] for it in kept[s]])
    arrays["open_loop_ctrl"] = OPEN_LOOP_CTRL
    arrays["open_loop_steps"] = OPEN_LOOP_STEPS
    arrays["beyond_target"] = BEYOND_TARGET
    arrays["beyond_steps"] = np.array(BEYOND_STEPS, np.int32)
    save_npz(OUT, arrays)


if __name__ == "__main__":
    main()
