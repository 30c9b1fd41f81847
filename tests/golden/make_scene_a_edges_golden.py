#!/usr/bin/env python
"""Generates tests/golden/scene_a_edges.npz: states of the 6-object scene (UR5gripper_2_finger.xml) chosen to take the warp-per-env
build of the engine to its capacity edges (tests/test_scene_a_edges_gpu.py).

TEST INFRASTRUCTURE.  All states come from the fp64 CPU oracle.  Scene A has one arm tree of 8 dofs and six 6-dof object trees
(box_1-3, ball_1-3), so the Newton Hessian needs Σ blocks = 162 doubles with every tree uncoupled, 210 / 294 / 414 with the arm and 1 / 2
/ 3 objects in one island, 378 / 522 / 702 for an island of 4 / 5 / 6 objects and 990 (the full triangle) for all seven trees.  The
engine's default region holds 410 doubles, the smallest one GE_HCAP accepts 336.  Resets scatter the objects, so big islands are built:
  * clusters placed on the table (source 0): a tower of the three boxes, each rotated 45 degrees about z against the one below (box-box
    faces clipped to octagons: 8 contact points), with 0-3 balls leaning against its foot or lying on top; all six objects packed in a
    corner of the drop bin.  A snapshot at placement and then every SETTLE_EVERY sub-steps while the arm holds HOME (balls roll off,
    the tower settles);
  * scripted grasp descents (source 1 descent, 2 closing) onto the tower, as tests/test_scene_b_gpu.py::test_scene_b_grasp_attempt_parity
    does: above it, rotate, open, descend, close, a snapshot every DESCENT_EVERY sub-steps; the fingers couple the arm to the tower;
  * closing snapshots with the three balls put against the tower's foot (source 3): the largest island, all seven trees;
  * single boxes jammed into a corner of the drop bin, against its floor and two walls (source 4): the most contacts on one tree that
    touches only static geometry.
Each snapshot is measured with one oracle forward(): contacts, and the contact graph over the kinematic trees (a contact between two
dynamic bodies of different trees couples them; the engine couples through ACTIVE contacts only, so the graph is an upper bound).
Block sum = Σ over components n (n + 1) / 2 + the uncoupled trees' own blocks.  Candidates are only states whose forward() agrees
within a tenth of the GPU tests' tolerances between the oracle and its -ffp-contract=fast build.  Only qpos / qvel and the metrics are
stored; the tests run the oracle's forward() themselves.

The .npz is written with fixed zip timestamps, so a rerun reproduces the committed file byte for byte.

  python tests/golden/make_scene_a_edges_golden.py      (under a minute)
"""
import io
import os
import sys
import zipfile
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "scene_a_edges.npz")
SETTLE_EVERY, SETTLE_TO = 25, 300
DESCENT_EVERY = 25
HCAP_MIN, HCAP_DEFAULT = 336, 410
MAXCON = 32
PEN = 5e-4  # built states: every placed contact starts 0.5 mm deep
TABLE = 0.91  # top of the pick table, centred at (0, -0.6)
BIN = (0.6, 0.1, 0.645, 0.2, 0.3)  # drop bin: centre x, y, floor top, inner half extents x, y
FIRST_OBJ_BODY = 18
BOX_HALF = {0: 0.02, 1: 0.015, 2: 0.025}  # box_1-3
BALL_R = {3: 0.03, 4: 0.025, 5: 0.02}  # ball_1-3
HOME = np.array([0, -1.57, 1.57, -1.57, -1.57, 0.0, 0.3])


def _scene():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    return load_scene_blob("A"), load_scene("A")[0]


def _quat_z(deg):
    a = np.radians(deg) / 2
    return np.array([np.cos(a), 0, 0, np.sin(a)])


def _base(A):
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(6):  # parked far apart on the floor's level, out of reach of everything
        _place(A, q, i, [2.0 + 0.3 * i, 2.0, 1.5])
    return q


def _place(A, q, i, world, quat=(1, 0, 0, 0)):
    """object i (0-2 box_1-3, 3-5 ball_1-3) with its centre at `world`: its free joint's qpos is relative to the body's position"""
    bp = np.asarray(A["body_pos"]).reshape(-1, 3)[FIRST_OBJ_BODY + i]
    q[8 + 7 * i:11 + 7 * i] = np.asarray(world) - bp
    q[11 + 7 * i:15 + 7 * i] = quat


def _tower(A, balls, x=0.0, y=-0.6):
    """box_3 on the table, box_1 on it turned 45 degrees, box_2 on box_1 turned back; `balls`: 'foot' (against box_3's faces, on
    the table), 'top' (ball_3 on box_2) or a number of foot balls"""
    q = _base(A)
    z = TABLE
    for i, turn in ((2, 0), (0, 45), (1, 0)):
        h = BOX_HALF[i]
        _place(A, q, i, [x, y, z + h - PEN], _quat_z(turn))
        z += 2 * h - PEN
    dirs = [(1, 0), (-1, 0), (0, 1)]
    for k in range(balls if isinstance(balls, int) else 0):
        r = BALL_R[3 + k]
        d = BOX_HALF[2] + r - PEN
        _place(A, q, 3 + k, [x + d * dirs[k][0], y + d * dirs[k][1], TABLE + r - PEN])
    if balls == "top":
        _place(A, q, 5, [x, y, z + BALL_R[5] - PEN])
    return q


def _bin_corner(A, which, packed):
    """box `which` in the drop bin's (-x, -y) corner on its floor against both walls; `packed`: the other five objects against it"""
    q = _base(A)
    bx, by, bz, hx, hy = BIN
    h = BOX_HALF[which]
    c = np.array([bx - hx + h - PEN, by - hy + h - PEN, bz + h - PEN])
    _place(A, q, which, c)
    if packed:
        others = [i for i in range(3) if i != which]
        x = c[0] + h
        for i in others:  # along +x from the corner box, each against the previous one and the -y wall
            hi = BOX_HALF[i]
            _place(A, q, i, [x + hi - PEN, by - hy + hi - PEN, bz + hi - PEN])
            x += 2 * hi - PEN
        y = c[1] + h
        for k in range(3):  # along +y from the corner box, against the -x wall
            r = BALL_R[3 + k]
            _place(A, q, 3 + k, [bx - hx + r - PEN, y + r - PEN, bz + r - PEN])
            y += 2 * r - PEN
    return q


def measure(o, A):
    """one forward() of the oracle on its state: contact count, contact-graph components over the trees, block sum, the largest
    number of contacts on one tree that no contact couples to another (the engine's 8-lane group path takes at most 15)"""
    from tests.common import contact_is_analytic

    o.forward()
    c = o.contacts()
    body_tree = _body_tree(A)
    gb = np.asarray(A["geom_bodyid"]).ravel()
    tdn = np.asarray(A["tree_dofnum"]).ravel()
    nt = len(tdn)
    parent = list(range(nt))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    trees = [(body_tree[gb[int(g1)]], body_tree[gb[int(g2)]]) for g1, g2 in c[:, 13:15]]
    coupled = np.zeros(nt, bool)
    for t1, t2 in trees:
        if t1 >= 0 and t2 >= 0 and t1 != t2:
            coupled[t1] = coupled[t2] = True
            a, b = find(t1), find(t2)
            parent[max(a, b)] = min(a, b)
    comp = {}
    for t in range(nt):
        if coupled[t]:
            comp.setdefault(find(t), []).append(t)
    sizes = sorted((int(tdn[m].sum()) for m in comp.values()), reverse=True)
    blocks = sum(n * (n + 1) // 2 for n in sizes) + sum(int(tdn[t]) * (int(tdn[t]) + 1) // 2 for t in range(nt) if not coupled[t])
    per_tree = np.zeros(nt, int)
    for t1, t2 in trees:
        for t in {t1, t2}:
            if t >= 0 and not coupled[t]:
                per_tree[t] += 1
    largest = max(comp.values(), key=lambda m: int(tdn[m].sum())) if comp else []
    nan = int(contact_is_analytic(A, c).sum()) if len(c) else 0
    return {"ncon": int(o.ncon), "ncomp": len(sizes), "largest": sizes[0] if sizes else 0, "largest_trees": len(largest),
            "blocks": int(blocks), "uncoupled_tree_max_contacts": int(per_tree.max()), "arm_in_largest": int(0 in largest),
            "ncand": int(o.ncand), "nanalytic": nan}


def _body_tree(A):
    lastdof = np.asarray(A["body_lastdof"]).ravel()
    dti = np.asarray(A["dof_treeindex"]).ravel()
    return np.array([-1 if d < 0 else int(dti[d]) for d in lastdof])


def _configs(A):
    """the placed clusters: (name, qpos)"""
    out = [("tower", _tower(A, 0)), ("tower+1 ball", _tower(A, 1)), ("tower+2 balls", _tower(A, 2)), ("tower+3 balls", _tower(A, 3)),
           ("tower+ball on top", _tower(A, "top"))]
    out += [("bin corner, box_%d" % (i + 1), _bin_corner(A, i, False)) for i in range(3)]
    out += [("bin corner, all packed", _bin_corner(A, 2, True))]
    return out


def settle_run(k):
    from oracle.oracle_py import OracleEnv

    blob, A = _scene()
    name, q = _configs(A)[k]
    o = OracleEnv(blob)
    o.reset(q)
    src = 4 if name.startswith("bin corner, box") else 0
    out = [({"source": src, "config": k, "step": 0}, q.copy(), np.zeros(44))]
    for step in range(SETTLE_EVERY, SETTLE_TO + 1, SETTLE_EVERY):
        o.move_group("All", HOME, 1e-9, SETTLE_EVERY)
        out.append(({"source": src, "config": k, "step": step}, o.qpos.copy(), o.qvel.copy()))
    o.close()
    return out


def descent_coords(A, q):
    """the grasp target of the tower runs: box_1 in the middle of the tower (it touches box_3 and box_2), 2 cm above its centre"""
    from tests.common import object_positions

    p = object_positions(A, q)[0]
    return np.array([p[0], p[1], p[2] + 0.02])


def descent_run(k):
    """GraspEnv.move_and_grasp's phases (GraspingEnv.py:205-386) up to the closed gripper on the tower of config k, the descent and
    the closing cut into movements of DESCENT_EVERY sub-steps; source 3: closing snapshots with the balls put against the tower"""
    from oracle.oracle_py import OracleEnv

    blob, A = _scene()
    o = OracleEnv(blob)
    o.reset(_configs(A)[k][1])
    coords = descent_coords(A, o.qpos)
    o.move_ee(np.array([coords[0], coords[1], 1.1]), 0.05, 1000)
    o.target[5] = 30 * np.pi / 180
    o.move_group("All", None, 0.05, 500)
    o.move_group("Gripper", np.array([0.0]), 0.05, 1000)
    out, step = [], 0
    c2 = np.array([coords[0], coords[1], max(coords[2] - 0.01, TABLE)])
    for phase, (tgt, tol, budget) in enumerate([(c2, 0.01, 300), (np.array([-0.4]), 0.01, 300)]):
        done = 0
        while done < budget:
            if phase == 0:
                r, s = o.move_ee(tgt, tol, DESCENT_EVERY)
            else:
                r, s = o.move_group("Gripper", tgt, tol, DESCENT_EVERY)
            assert r in (1, 2), "no IK solution for the descent target"
            done += s - 1
            step += s - 1
            q, v = o.qpos.copy(), o.qvel.copy()
            out.append(({"source": 1 + phase, "config": k, "step": step}, q, v))
            if phase == 1:  # the balls against the tower's foot, on the table, at rest
                qb = q.copy()
                vb = v.copy()
                _balls_at_foot(A, qb)
                vb[26:44] = 0
                out.append(({"source": 3, "config": k, "step": step}, qb, vb))
            if r == 1:
                break
        if phase == 0:
            o.stay(100)
    o.close()
    return out


def _balls_at_foot(A, q):
    """the three balls against box_3's faces (its own frame: +x, -x, +y), lying on the table"""
    from tests.common import object_positions

    p = object_positions(A, q)[2]
    w, x, y, z = q[8 + 7 * 2 + 3:8 + 7 * 2 + 7]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    for k, d in enumerate([(1, 0, 0), (-1, 0, 0), (0, 1, 0)]):
        r = BALL_R[3 + k]
        c = p + R @ (np.array(d) * (BOX_HALF[2] + r - PEN))
        c[2] = TABLE + r - PEN
        _place(A, q, 3 + k, c)


def measure_all(args):
    """metrics of each state, and its contacts / qacc (`so`: the oracle build)"""
    items, so = args
    if so:
        os.environ["GRASP_ORACLE_SO"] = so
    from oracle.oracle_py import OracleEnv

    blob, A = _scene()
    o = OracleEnv(blob)
    res = []
    for tag, q, v in items:
        o.reset(q, v)
        res.append((measure(o, A), o.contacts(), o.field("qacc")))
    o.close()
    return res


def robust(a, b, A):
    """the same forward() on two oracle builds agrees within a tenth of the GPU tests' tolerances (analytic contacts 1e-10, MPR
    contacts 1e-8, qacc 1e-7 x scale)"""
    from tests.common import contact_is_analytic

    (_, ca, qa), (_, cb, qb) = a, b
    if ca.shape != cb.shape or not np.array_equal(ca[:, 13:], cb[:, 13:]):
        return False
    if len(ca):
        tol = np.where(contact_is_analytic(A, ca), 1e-10, 1e-8)
        if (np.abs(ca[:, :13] - cb[:, :13]).max(axis=1) >= tol).any():
            return False
    return np.abs(qa - qb).max() <= 1e-7 * max(1.0, float(np.abs(qa).max()))


def select(tags, mets):
    """indices of the kept states and why each was kept"""
    chosen, why = [], {}

    def take(i, reason):
        if i not in chosen:
            chosen.append(i)
            why[i] = []
        why[i].append(reason)

    n = len(mets)
    col = {k: np.array([m[k] for m in mets]) for k in mets[0]}
    # (a) block sums that fit the default region and overflow the minimum one: one per kind of island first
    band_a = [i for i in range(n) if HCAP_MIN < mets[i]["blocks"] <= HCAP_DEFAULT]
    seen = set()
    for i in sorted(band_a, key=lambda i: (-mets[i]["ncon"], i)):
        key = (mets[i]["blocks"], tags[i]["config"])
        if key not in seen and len(seen) < 3:
            seen.add(key)
            take(i, "block sum %d in (%d, %d]" % (mets[i]["blocks"], HCAP_MIN, HCAP_DEFAULT))
    # (b) just above the default region
    band_b = [i for i in range(n) if HCAP_DEFAULT < mets[i]["blocks"] <= 480]
    for i in sorted(band_b, key=lambda i: (mets[i]["blocks"], -mets[i]["ncon"], i))[:2]:
        take(i, "block sum %d just above %d" % (mets[i]["blocks"], HCAP_DEFAULT))
    # (c) the largest island
    top = col["largest"].max()
    for i in sorted((i for i in range(n) if col["largest"][i] == top), key=lambda i: (-mets[i]["ncon"], i))[:2]:
        take(i, "largest island (%d trees, %d dofs, block sum %d)" % (mets[i]["largest_trees"], top, mets[i]["blocks"]))
    # (d) the most contacts, analytic and MPR mixed
    mixed = [i for i in range(n) if 0 < mets[i]["nanalytic"] < mets[i]["ncon"]]
    i = max(mixed, key=lambda i: (mets[i]["ncon"], -i))
    take(i, "most contacts (%d: %d analytic, %d MPR)" % (mets[i]["ncon"], mets[i]["nanalytic"], mets[i]["ncon"] - mets[i]["nanalytic"]))
    i = max(mixed, key=lambda i: (mets[i]["ncon"] - mets[i]["nanalytic"], mets[i]["ncon"], -i))
    take(i, "most MPR contacts (%d of %d)" % (mets[i]["ncon"] - mets[i]["nanalytic"], mets[i]["ncon"]))
    # a capacity that ends inside the analytic contacts without cutting the candidate list (2 maxcon >= ncand, maxcon >= 16)
    room = [m["nanalytic"] - max(16, (m["ncand"] + 1) // 2) for m in mets]
    i = int(np.argmax(room))
    take(i, "%d analytic contacts, %d candidates" % (mets[i]["nanalytic"], mets[i]["ncand"]))
    # (e) the most contacts on one tree that touches static geometry only
    i = int(col["uncoupled_tree_max_contacts"].argmax())
    take(i, "%d contacts on one uncoupled tree" % col["uncoupled_tree_max_contacts"].max())
    # a settling cluster with many islands
    i = max(range(n), key=lambda i: (mets[i]["ncomp"], mets[i]["ncon"], -i))
    take(i, "%d contact-graph components" % mets[i]["ncomp"])
    return chosen, why


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
    import subprocess

    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "fast"])
    fast = os.path.join(ROOT, "oracle", "libgrasp_oracle_fast.so")
    blob, A = _scene()
    names = [c[0] for c in _configs(A)]
    towers = [k for k, nm in enumerate(names) if nm in ("tower", "tower+1 ball")]
    with Pool(min(8, os.cpu_count() or 1), maxtasksperchild=1) as pool:
        runs = pool.map(settle_run, range(len(names))) + pool.map(descent_run, towers)
        items = [it for r in runs for it in r]
        res = {}
        for so in (None, fast):
            out = pool.map(measure_all, [(items[c::8], so) for c in range(8)], chunksize=1)
            res[so] = [out[i % 8][i // 8] for i in range(len(items))]
    ok = [robust(res[None][i], res[fast][i], A) for i in range(len(items))]
    allm = [r[0] for r in res[None]]
    print("%d snapshots measured, %d rounding-sensitive ones dropped" % (len(items), ok.count(False)))
    print("over all snapshots: at most %d contacts (%d above the default capacity %d), %d candidates; largest island %d trees / %d "
          "dofs; at most %d contacts on one uncoupled tree (the group path takes 15)" % (
              max(m["ncon"] for m in allm), sum(m["ncon"] > MAXCON for m in allm), MAXCON, max(m["ncand"] for m in allm),
              max(m["largest_trees"] for m in allm), max(m["largest"] for m in allm), max(m["uncoupled_tree_max_contacts"] for m in allm)))
    print("block sums reached:", sorted({m["blocks"] for m in allm}))
    items = [it for it, k in zip(items, ok) if k]
    mets = [r[0] for r, k in zip(res[None], ok) if k]
    tags = [t for t, _, _ in items]
    chosen, why = select(tags, mets)
    for i in chosen:
        t, m = tags[i], mets[i]
        print("%-7s %-24s step %4d: ncon %2d (%2d analytic)  ncand %2d  components %d  largest %d trees / %2d dofs  block sum %3d  "
              "-- %s" % (["cluster", "descent", "closing", "balls", "corner"][t["source"]], names[t["config"]], t["step"], m["ncon"],
                          m["nanalytic"], m["ncand"], m["ncomp"], m["largest_trees"], m["largest"], m["blocks"], "; ".join(why[i])))
    arrays = {"qpos": np.array([items[i][1] for i in chosen]), "qvel": np.array([items[i][2] for i in chosen])}
    for k in ("source", "config", "step"):
        arrays[k] = np.array([tags[i][k] for i in chosen], np.int32)
    for k in mets[0]:
        arrays[k] = np.array([mets[i][k] for i in chosen], np.int32)
    save_npz(OUT, arrays)


if __name__ == "__main__":
    main()
