#!/usr/bin/env python
"""Generates tests/golden/scene_a1.npz (+ scene_a1.json, a readable summary): states and grasp attempts of scene A1, the 6-object
scene with every object turned into the 4 cm cube of box_1 (model/scene.py: _equal_size_objects), for tests/test_scene_a1_gpu.py.

TEST INFRASTRUCTURE.  Everything comes from the fp64 CPU oracle.  A1's cubes start at body heights 0.95 .. 1.5 m with identity
orientation, so in a large share of resets one cube falls onto another: two equal, exactly axis-aligned boxes meet, their face-axis
SAT separations tie bit for bit (the strict `>` of col_box_box picks the reference box), the edge axes are parallel (skipped by the
1e-6 guard) and two equal squares are clipped against each other.  Stored:
  * resets (env i of episode 0 = RandomState(20000 + i), settled by stay(1000) in its 50 chunks): the final pose of seeds 0..N_RESET-1
    from the oracle and from its -ffp-contract=fast build, each cube's outcome (which body axis points up, tilt, resting on the table
    or on a cube) and whether a cube fell onto another; for seeds of every outcome kind (flip by 90 / 180 degrees, tilted, stacked)
    the state at reset, at the first cube-cube contact, during the tumble and at rest;
  * hand-built equal-cube states, each tagged with the col_box_box branch it is built for (TAGS);
  * grasp attempts as GraspEnv.step runs them (depth at the action pixel -> pixel_2_world -> move_and_grasp), aimed at cube centres:
    8 consecutive attempts of each of N_EPISODES environments (cubes pile up in the drop bin); every record keeps the state before it;
  * a tie / rounding probe per state: the contact list's signature (count, geom pairs, and per box-box pair the outcome, reference
    box and points kept) with each cube moved by +-1e-13 m along each world axis, and on the fast build.  A state whose signature
    changes is rounding-decided ("flag"); the other lists are stored as alternatives.  Other states are kept only if forward()
    agrees between the two builds within a tenth of the GPU tests' tolerances;
  * contact counts: ncon of every state, the most contacts one collision stage found during a settle or an attempt (uncapped), and
    whether the attempt's outcome is unchanged with the oracle capped at the engine's 32 contacts.
The .npz is written with fixed zip timestamps, so a rerun reproduces the committed file byte for byte.

  python tests/golden/make_scene_a1_golden.py      (about a minute on 8 cores)
"""
import io
import json
import os
import sys
import zipfile
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "scene_a1")
N_RESET = 200
SEED_BASE = 20000
ATTEMPT_ENVS = list(range(100, 116))  # 16 environments x 8 attempts
N_STEPS, W, H, TABLE_HEIGHT = 8, 200, 200, 0.91
N_EPISODES = 4
MAXCON = 32
H_CUBE = 0.02
PEN = 5e-4
TABLE = 0.91
BIN = (0.6, 0.1, 0.645, 0.2, 0.3)  # drop bin: centre x, y, floor top, inner half extents x, y
FIRST_OBJ_BODY, FIRST_CUBE_GEOM = 18, 30
EPS_MOVE = 1e-13
HOME = np.array([0, -1.57, 1.57, -1.57, -1.57, 0.0, 0.3])
TAGS = ["stack aligned", "stack offset x", "stack offset xy", "side by side", "stack rotated 1e-9", "bin wall stack", "held above cube"]
KINDS = ["reset", "first contact", "tumble", "rest", "built"]
# centre of the built stacks: at x = 0, x +- h is exact in fp64, so equal cubes with the same x have x faces that coincide bit for
# bit and incident vertices exactly on the reference face's clip lines (no other table coordinate has that property for h = 0.02)
X0, Y0 = 0.0, -0.5


def _scene():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    return load_scene_blob("A1"), load_scene("A1")[0]


def _use_build(so):
    """pool initializer: the worker loads the oracle build `so` (the library is loaded once per process)"""
    os.environ["GRASP_ORACLE_SO"] = so


def _oracle(blob):
    from oracle.oracle_py import OracleEnv

    return OracleEnv(blob)


def reset_qpos(A, i):
    from mujoco_rl_ur5_b200.batched_env import scene_a_reset_qpos

    return scene_a_reset_qpos(A, SEED_BASE + i)


def quat_mat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def outcome(A, q):
    """per cube: the body axis pointing up (+-1..3), its tilt from the vertical in degrees, 1 if it rests on another cube"""
    from tests.common import object_positions

    p = object_positions(A, q)
    up, tilt, on = [], [], []
    for i in range(6):
        R = quat_mat(q[11 + 7 * i:15 + 7 * i] / np.linalg.norm(q[11 + 7 * i:15 + 7 * i]))
        k = int(np.abs(R[2]).argmax())
        up.append(int(np.sign(R[2, k])) * (k + 1))
        tilt.append(float(np.degrees(np.arccos(min(1.0, abs(R[2, k]))))))
        below = [j for j in range(6) if j != i and np.hypot(*(p[i, :2] - p[j, :2])) < 0.045 and p[j, 2] < p[i, 2] - 0.02]
        on.append(int(bool(below) and p[i, 2] > TABLE + 1.5 * 2 * H_CUBE - 0.01))
    return np.array(up), np.array(tilt), np.array(on)


def cube_cube_contacts(o):
    bb = o.boxbox()
    return int(sum(r[8] for r in bb if r[0] >= FIRST_CUBE_GEOM and r[1] >= FIRST_CUBE_GEOM))


def reset_run(i):
    """stay(1000) from reset i as its 50 chunks: final qpos, chunk of the first cube-cube contact, snapshots, peak ncon"""
    blob, A = _scene()
    o = _oracle(blob)
    q0 = reset_qpos(A, i)
    o.reset(q0)
    o.ncon_peak(True)
    snaps, first = [(0, q0.copy(), np.zeros(o.nv))], -1
    for c in range(50):
        o.move_group("All", None, 1e-7, 10)
        if first < 0 and cube_cube_contacts(o):
            first = c
            snaps.append((1, o.qpos.copy(), o.qvel.copy()))
        if first >= 0 and c == first + 4:
            snaps.append((2, o.qpos.copy(), o.qvel.copy()))
    snaps.append((3, o.qpos.copy(), o.qvel.copy()))
    o.forward()
    res = {"qpos": o.qpos.copy(), "first": first, "peak": o.ncon_peak(True), "ncon": int(o.ncon), "snaps": snaps}
    o.close()
    return res


def _place(A, q, i, world, quat=(1, 0, 0, 0)):
    bp = np.asarray(A["body_pos"]).reshape(-1, 3)[FIRST_OBJ_BODY + i]
    q[8 + 7 * i:11 + 7 * i] = np.asarray(world) - bp
    q[11 + 7 * i:15 + 7 * i] = quat


def _base(A):
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(6):  # parked far apart, out of reach of everything
        _place(A, q, i, [2.0 + 0.3 * i, 2.0, 1.5])
    return q


def built_states(blob, A):
    """(tag index, qpos, qvel) of the hand-built states"""
    h, z0 = H_CUBE, TABLE + H_CUBE - PEN
    z1 = z0 + 2 * H_CUBE - PEN
    out = []

    def stack(dx, dy, quat=(1, 0, 0, 0)):
        q = _base(A)
        _place(A, q, 0, [X0, Y0, z0])
        _place(A, q, 1, [X0 + dx, Y0 + dy, z1], quat)
        return q

    out.append((0, stack(0, 0)))
    out.append((1, stack(h, 0)))
    out.append((2, stack(h, h)))
    q = _base(A)
    _place(A, q, 0, [X0, Y0, z0])
    _place(A, q, 1, [X0, Y0 + 2 * h - PEN, z0])
    out.append((3, q))
    e = 0.5e-9
    out.append((4, stack(0, 0, (np.cos(e), 0, 0, np.sin(e)))))
    bx, by, bz, hx, hy = BIN
    q = _base(A)
    _place(A, q, 0, [bx - hx + h - PEN, by, bz + h - PEN])
    _place(A, q, 1, [bx - hx + h - PEN, by, bz + 3 * h - 2 * PEN])
    out.append((5, q))
    out.append((6, held_above_cube(blob, A)))
    return [(t, q, np.zeros(len(A["qpos0"]) - 6)) for t, q in out]


def held_above_cube(blob, A):
    """box_1 grasped from the table and lifted (the descent / closing phases of move_and_grasp), then box_2 put under it, its top
    0.5 mm into the held cube's lowest point"""
    from tests.common import object_positions

    q = _base(A)
    _place(A, q, 0, [X0, -0.6, TABLE + H_CUBE - PEN])
    o = _oracle(blob)
    o.reset(q)
    o.stay(200)
    p = object_positions(A, o.qpos)[0]
    o.move_ee(np.array([p[0], p[1], 1.1]), 0.05, 1000)
    o.move_group("Gripper", np.array([0.0]), 0.05, 1000)
    o.move_ee(np.array([p[0], p[1], p[2] - 0.01]), 0.01, 300)
    o.stay(100)
    o.move_group("Gripper", np.array([-0.4]), 0.01, 300)
    o.move_ee(np.array([p[0], p[1], 1.0]), 0.01, 600)
    q = o.qpos.copy()
    o.close()
    c = object_positions(A, q)[0]
    R = quat_mat(q[11:15])
    low = c[2] - np.abs(R[2]).sum() * H_CUBE
    _place(A, q, 1, [c[0], c[1], low - H_CUBE + PEN])
    return q


def signature(o):
    c = o.contacts()
    bb = o.boxbox()
    return (int(o.ncon), tuple(map(tuple, c[:, 13:15].astype(int).tolist())),
            tuple(tuple(int(v) for v in r[[0, 1, 2, 3, 8]]) for r in bb if r[2] > 0))


def probe(args):
    """forward() of one state: [(signature, contacts, qacc, qfrc_constraint, boxbox, ncon)], the state itself first, then (moves)
    with every cube moved by +-EPS_MOVE along each world axis"""
    q, v, moves = args
    blob, A = _scene()
    o = _oracle(blob)
    r = []
    for mv in [None] + ([(i, ax, sgn) for i in range(6) for ax in range(3) for sgn in (1, -1)] if moves else []):
        qq = q.copy()
        if mv:
            i, ax, sgn = mv
            qq[8 + 7 * i + ax] += sgn * EPS_MOVE
        o.reset(qq, v)
        o.forward()
        r.append((signature(o), o.contacts(), o.field("qacc"), o.field("qfrc_constraint"), o.boxbox(), int(o.ncon)))
    o.close()
    return r


def robust(a, b, A):
    """the same forward() on two oracle builds agrees within a tenth of the GPU tests' tolerances"""
    from tests.common import contact_is_analytic

    ca, qa, fa = a[1], a[2], a[3]
    cb, qb, fb = b[1], b[2], b[3]
    if ca.shape != cb.shape or not np.array_equal(ca[:, 13:], cb[:, 13:]):
        return False
    if len(ca):
        tol = np.where(contact_is_analytic(A, ca), 1e-10, 1e-8)
        if (np.abs(ca[:, :13] - cb[:, :13]).max(axis=1) >= tol).any():
            return False
    return all(np.abs(x - y).max() <= 1e-7 * max(1.0, float(np.abs(x).max())) for x, y in ((qa, qb), (fa, fb)))


def attempt_env(i):
    """N_STEPS consecutive GraspEnv.step attempts of environment i, each aimed at the centre of a cube lying in the camera's view"""
    from tests.common import object_positions

    blob, A = _scene()
    cam = int(np.asarray(A["cam_top_down"]).ravel()[0])
    o = _oracle(blob)
    o.reset(reset_qpos(A, i))
    o.stay(1000)
    rng = np.random.RandomState(40000 + i)
    rec = []
    for k in range(N_STEPS):
        q, v = o.qpos.copy(), o.qvel.copy()
        o.reset(q, v)
        _, depth = o.render(cam, W, H)
        ys, xs = np.where((depth < 1.09 - 0.005) & (depth > 1.09 - 0.1))
        p = object_positions(A, q)
        cubes = [j for j in range(6) if p[j, 1] < -0.3 and TABLE < p[j, 2] < 1.1]
        if not cubes or not len(ys):
            break
        j = cubes[rng.randint(len(cubes))]
        world = np.array([o.pixel_2_world(x, y, depth[y, x], cam, W, H) for y, x in zip(ys, xs)])
        best = int(np.argmin(np.hypot(world[:, 0] - p[j, 0], world[:, 1] - p[j, 1])))
        x, y = int(xs[best]), int(ys[best])
        a = [y * W + x, int(rng.randint(0, 6))]
        d = float(depth[y][x])
        c = o.pixel_2_world(x, y, d, cam, W, H)
        executed = not (c[2] < 0.8 or c[1] > -0.3)
        o.ncon_peak(True)
        reward, info = o.move_and_grasp(c, a[1], TABLE_HEIGHT) if executed else (0, [0] * 12)
        peak = o.ncon_peak(True)
        q1 = o.qpos.copy()
        capped = _oracle(blob)  # the same attempt with the engine's 32-contact list
        capped.set_maxcon(MAXCON)
        capped.reset(q, v)
        r32, i32 = capped.move_and_grasp(c, a[1], TABLE_HEIGHT) if executed else (0, [0] * 12)
        same = (r32, i32) == (reward, info) and np.array_equal(capped.qpos, q1)
        capped.close()
        rec.append({"env": i, "step": k, "action": a, "depth": d, "coords": [float(t) for t in c], "executed": int(executed),
                    "reward": int(reward), "info": [int(t) for t in info], "arm_qpos": q1[:8].copy(), "q0": q, "v0": v,
                    "peak": peak, "cap32_same": int(same), "target": j})
    o.close()
    return rec


def save_npz(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member (np.savez stamps the current time)"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def reset_kind(up, tilt, on, moved):
    """outcome kinds of one settled reset, over the cubes that took part in a cube-cube fall"""
    kinds = set()
    for i in np.flatnonzero(moved):
        if on[i]:
            kinds.add("stacked")
        if tilt[i] > 5:
            kinds.add("tilted")
        elif abs(up[i]) != 3:
            kinds.add("flip 90")
        elif up[i] == -3:
            kinds.add("flip 180")
    return kinds


def main():
    import subprocess

    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "fast"])
    fast = os.path.join(ROOT, "oracle", "libgrasp_oracle_fast.so")
    blob, A = _scene()
    nv = len(A["qpos0"]) - 6
    ncpu = min(8, os.cpu_count() or 1)
    with Pool(ncpu) as pool, Pool(ncpu, initializer=_use_build, initargs=(fast,)) as pool_fast:
        resets = pool.map(reset_run, range(N_RESET))
        resets_fast = pool_fast.map(reset_run, range(N_RESET))
        attempts = [r for e in pool.map(attempt_env, ATTEMPT_ENVS) for r in e]
        built = built_states(blob, A)

        # reset outcomes on both builds
        R = {k: [] for k in ("up", "tilt", "on", "up_fast", "on_fast", "fell", "robust", "peak", "ncon")}
        kinds_by_seed = []
        for i, (r, rf) in enumerate(zip(resets, resets_fast)):
            up, tilt, on = outcome(A, r["qpos"])
            upf, _, onf = outcome(A, rf["qpos"])
            cubes = np.concatenate([np.arange(8 + 7 * j, 15 + 7 * j) for j in range(6)])
            R["up"].append(up); R["tilt"].append(tilt); R["on"].append(on); R["up_fast"].append(upf); R["on_fast"].append(onf)
            R["fell"].append(int(r["first"] >= 0)); R["peak"].append(r["peak"]); R["ncon"].append(r["ncon"])
            R["robust"].append(int(np.abs(r["qpos"][cubes] - rf["qpos"][cubes]).max() < 1e-8))
            p0 = reset_qpos(A, i)
            moved = [abs(tilt[j]) > 1 or np.abs(r["qpos"][8 + 7 * j:10 + 7 * j] - p0[8 + 7 * j:10 + 7 * j]).max() > 0.005 for j in range(6)]
            kinds_by_seed.append(reset_kind(up, tilt, on, moved) if r["first"] >= 0 else set())
        # seeds whose snapshots are stored: the first two of every outcome kind
        chosen = []
        for kind in ("flip 90", "flip 180", "tilted", "stacked"):
            for i in [i for i in range(N_RESET) if kind in kinds_by_seed[i]][:2]:
                if i not in chosen:
                    chosen.append(i)
        items = [(KINDS.index(KINDS[k]), i, -1, q, v) for i in chosen for k, q, v in resets[i]["snaps"]]
        items += [(4, -1, t, q, v) for t, q, v in built]
        n = len(items)
        pr = pool.map(probe, [(it[3], it[4], True) for it in items])
        prf = pool_fast.map(probe, [(it[3], it[4], False) for it in items])

    keep, flags, alts, report = [], [], [], []
    for s in range(n):
        base = pr[s][0]
        variants = pr[s][1:] + prf[s]
        sigs = {}
        for var in variants:
            if var[0] != base[0] and var[0] not in sigs:
                sigs[var[0]] = var
        flag = int(bool(sigs))
        ok = flag or robust(base, prf[s][0], A)
        report.append((KINDS[items[s][0]], items[s][1], TAGS[items[s][2]] if items[s][2] >= 0 else "", base[5], flag, ok))
        if not ok:
            continue
        keep.append(s)
        flags.append(flag)
        alts.append(list(sigs.values()))
    for r in report:
        print("%-13s seed %3d %-20s ncon %2d  rounding-decided %d  kept %d" % r)
    S = len(keep)
    arrays = {"state_qpos": np.array([items[s][3] for s in keep]), "state_qvel": np.array([items[s][4] for s in keep]),
              "state_kind": np.array([items[s][0] for s in keep], np.int32), "state_seed": np.array([items[s][1] for s in keep], np.int32),
              "state_tag": np.array([items[s][2] for s in keep], np.int32), "state_flag": np.array(flags, np.int32),
              "state_ncon": np.array([pr[s][0][5] for s in keep], np.int32),
              "state_settle_peak": np.array([resets[items[s][1]]["peak"] if items[s][1] >= 0 else pr[s][0][5] for s in keep], np.int32)}
    alt_state, alt_con, alt_n, alt_qacc, alt_qfrc = [], [], [], [], []
    for k, a in enumerate(alts):
        for var in a:
            alt_state.append(k); alt_n.append(var[5]); alt_con.append(var[1]); alt_qacc.append(var[2]); alt_qfrc.append(var[3])
    arrays["alt_state"] = np.array(alt_state, np.int32)
    arrays["alt_ncon"] = np.array(alt_n, np.int32)
    arrays["alt_contacts"] = np.concatenate(alt_con) if alt_con else np.zeros((0, 16))
    arrays["alt_qacc"] = np.array(alt_qacc) if alt_qacc else np.zeros((0, nv))
    arrays["alt_qfrc_constraint"] = np.array(alt_qfrc) if alt_qfrc else np.zeros((0, nv))
    arrays["reset_qpos"] = np.array([r["qpos"] for r in resets])
    arrays["reset_qpos_fast"] = np.array([r["qpos"] for r in resets_fast])
    for k in R:
        arrays["reset_" + k] = np.array(R[k], np.float64 if k == "tilt" else np.int32)
    for k in ("q0", "v0", "coords", "action", "reward", "info", "arm_qpos", "depth", "env", "step", "executed", "peak", "cap32_same", "target"):
        arrays["att_" + k] = np.array([r[k] for r in attempts], np.float64 if k in ("q0", "v0", "coords", "arm_qpos", "depth") else np.int32)
    envs = [e for e in ATTEMPT_ENVS if sum(r["env"] == e for r in attempts) == N_STEPS][:N_EPISODES]
    arrays["episode_env"] = np.array(envs, np.int32)
    save_npz(OUT + ".npz", arrays)

    kinds = {k: [i for i in range(N_RESET) if k in kinds_by_seed[i]] for k in ("flip 90", "flip 180", "tilted", "stacked")}
    summary = {
        "about": "scene A1 (six 4 cm cubes) states and grasp attempts on the fp64 CPU oracle (tests/golden/make_scene_a1_golden.py)",
        "tags": TAGS, "kinds": KINDS,
        "resets": {"seeds": N_RESET, "cube_on_cube_falls": int(sum(R["fell"])), "both_builds_agree": int(sum(R["robust"])),
                   "outcome_kinds": {k: len(v) for k, v in kinds.items()}, "stored_seeds": chosen,
                   "ncon_at_rest_max": int(max(R["ncon"])), "ncon_settle_peak_max": int(max(R["peak"]))},
        "states": {"stored": S, "rounding_decided": int(sum(flags)), "alternatives": len(alt_state),
                   "dropped_not_robust": n - S},
        "attempts": {"records": len(attempts), "rewarded": int(sum(r["reward"] for r in attempts)),
                     "executed": int(sum(r["executed"] for r in attempts)), "episodes": envs,
                     "ncon_peak_max": int(max(r["peak"] for r in attempts)),
                     "ncon_peak_above_32": int(sum(r["peak"] > MAXCON for r in attempts)),
                     "changed_by_32_cap": int(sum(1 - r["cap32_same"] for r in attempts))},
    }
    with open(OUT + ".json", "w") as f:
        json.dump(summary, f, indent=1)
        f.write("\n")
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
