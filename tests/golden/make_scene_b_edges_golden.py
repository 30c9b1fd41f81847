#!/usr/bin/env python
"""Generates tests/golden/scene_b_edges.npz: states of the reference's default 40-object scene (UR5gripper_2_finger_many_objects.xml)
chosen to take the CTA-per-env build of the engine to its capacity edges (tests/test_scene_b_edges_gpu.py).

TEST INFRASTRUCTURE.  All states come from the fp64 CPU oracle:
  * resets by the live rule of GraspingEnv.py:418-430 with RandomState(20000 + seed), seeds 0-7, while the arm holds a set-point near
    HOME; a snapshot every 50 sub-steps up to 1200 (objects falling, impacts, piles forming and settling);
  * the scripted descent of tests/test_scene_b_gpu.py::test_scene_b_grasp_attempt_parity (seed 0, 499 settle sub-steps, the object
    nearest the table centre, rotation 1): move above it, rotate, open, descend, close - a snapshot every 25 sub-steps of the descent
    and of the closing, where the arm and the objects under the fingers form one island.
Each snapshot is measured with one oracle forward(): contacts, and the contact graph over the kinematic trees (a contact between two
dynamic bodies of different trees couples them).  Its components are the largest islands the engine can form (the engine couples trees
through ACTIVE contacts only, so the graph is an upper bound).  Per-state block sum = Σ over components n (n + 1) / 2 + the uncoupled
trees' own blocks, in doubles: what the Newton Hessian of that build needs if every contact is active.

Selection (about 12 states, printed with the reason): most contacts; most components; largest component in dofs; the largest block sum
(and whether it exceeds 2722 doubles, the engine's default Hessian region for this scene); further states with a component of >= 42 dofs
(an island that large overflows the minimum region Σ tree blocks + 6·112 + 64); descent / closing states with the arm in the largest
component; the state with the most analytic contacts beyond half its broad-phase candidates (a contact capacity can end inside the
analytic contacts without cutting the candidate list); the earliest snapshot with contacts (small candidate lists).  Candidates are
only states whose forward() agrees within a tenth of the GPU tests' tolerances between the oracle and its -ffp-contract=fast build: on
a rounding-sensitive state (seen: an MPR contact normal that moves by 2.6e-5) no build can be held to the oracle.  Only qpos / qvel
and the metrics are stored; the tests run the oracle's forward() themselves.

The .npz is written with fixed zip timestamps, so a rerun reproduces the committed file byte for byte.

  python tests/golden/make_scene_b_edges_golden.py      (about a minute on 8 cores: the oracle does ~100 sub-steps/s on this scene)
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
OUT = os.path.join(HERE, "scene_b_edges.npz")
SEEDS = range(8)
SETTLE_EVERY, SETTLE_TO = 50, 1200
DESCENT_EVERY = 25
HCAP_DEFAULT = 2722
BIG_ISLAND = 42
N_SELECT = 12
SETTLE_TARGET = np.array([0.2, 0.1, -0.1, 0.1, 0.1, 0.3, -0.1])  # offset from HOME, as tests/test_scene_b_gpu.py's settled states


def _scene():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    return load_scene_blob("B"), load_scene("B")[0]


def measure(o, A):
    """one forward() of the oracle on its state: contact count, contact-graph components over the trees, block sum, and the largest
    number of contacts on one tree that no contact couples to another (the engine's 8-lane group path takes at most 15)"""
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
    arm_in_largest = bool(comp) and 0 in max(comp.values(), key=lambda m: int(tdn[m].sum()))
    from tests.common import contact_is_analytic

    return {"ncon": int(o.ncon), "ncomp": len(sizes), "largest": sizes[0] if sizes else 0, "blocks": int(blocks),
            "uncoupled_tree_max_contacts": int(per_tree.max()), "arm_in_largest": int(arm_in_largest), "ncand": int(o.ncand),
            "nanalytic": int(contact_is_analytic(A, c).sum()) if len(c) else 0}


def _body_tree(A):
    lastdof = np.asarray(A["body_lastdof"]).ravel()
    dti = np.asarray(A["dof_treeindex"]).ravel()
    return np.array([-1 if d < 0 else int(dti[d]) for d in lastdof])


def settle_run(seed):
    from oracle.oracle_py import OracleEnv
    from tests.common import HOME, reset_qpos_scene_b

    blob, A = _scene()
    o = OracleEnv(blob)
    o.reset(reset_qpos_scene_b(A, seed))
    out = []
    for step in range(SETTLE_EVERY, SETTLE_TO + 1, SETTLE_EVERY):
        o.move_group("All", HOME + SETTLE_TARGET, 1e-7, SETTLE_EVERY)
        q, v = o.qpos.copy(), o.qvel.copy()
        out.append(({"source": 0, "seed": seed, "step": step}, q, v))
    o.close()
    return out


def descent_run(_):
    """tests/test_scene_b_gpu.py::test_scene_b_grasp_attempt_parity's attempt up to the closed gripper, with the descent and the
    closing cut into movements of DESCENT_EVERY sub-steps (GraspEnv.move_and_grasp's phases, GraspingEnv.py:205-386)"""
    from oracle.oracle_py import OracleEnv
    from tests.common import HOME, reset_qpos_scene_b

    blob, A = _scene()
    o = OracleEnv(blob)
    o.reset(reset_qpos_scene_b(A, 0))
    o.move_group("All", HOME + np.array([0, 0, 0, 0, 0, 0, 0.001]), 1e-9, 499)
    q = o.qpos.copy()
    pos = q[8:288].reshape(40, 7)[:, :3]
    on_table = (pos[:, 2] > 0.85) & (pos[:, 2] < 1.0)
    k = int((np.linalg.norm(pos[:, :2] - np.array([0.0, -0.6]), axis=1) + (~on_table) * 10).argmin())
    coords = np.array([pos[k, 0], pos[k, 1], pos[k, 2] + 0.02])
    o.move_ee(np.array([coords[0], coords[1], 1.1]), 0.05, 1000)
    o.target[5] = 30 * np.pi / 180
    o.move_group("All", None, 0.05, 500)
    o.move_group("Gripper", np.array([0.0]), 0.05, 1000)
    out, step = [], 0
    c2 = np.array([coords[0], coords[1], max(coords[2] - 0.01, 0.91)])
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
            out.append(({"source": 1 + phase, "seed": 0, "step": step}, o.qpos.copy(), o.qvel.copy()))
            if r == 1:
                break
        if phase == 0:
            o.stay(100)
    o.close()
    return out


def measure_all(args):
    """metrics of each state, and its contacts / qacc (`so`: the oracle build, as in make_scene_b_golden.py)"""
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


def robust(a, b):
    """the same forward() on two oracle builds agrees within the GPU tests' tolerances (contacts 1e-8, qacc 1e-7 x scale: a tenth of
    what the tests allow)"""
    (_, ca, qa), (_, cb, qb) = a, b
    if ca.shape != cb.shape or not np.array_equal(ca[:, 13:], cb[:, 13:]):
        return False
    return np.abs(ca[:, :13] - cb[:, :13]).max(initial=0.0) < 1e-8 and np.abs(qa - qb).max() <= 1e-7 * max(1.0, float(np.abs(qa).max()))


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
    take(int(col["ncon"].argmax()), "most contacts (%d)" % col["ncon"].max())
    take(int(col["ncomp"].argmax()), "most contact-graph components (%d)" % col["ncomp"].max())
    take(int(col["largest"].argmax()), "largest component (%d dofs)" % col["largest"].max())
    take(int(col["blocks"].argmax()), "largest block sum (%d doubles, %s the default region of %d)" % (
        col["blocks"].max(), "exceeds" if col["blocks"].max() > HCAP_DEFAULT else "within", HCAP_DEFAULT))
    arm = [i for i in range(n) if tags[i]["source"] > 0 and mets[i]["arm_in_largest"]]
    for i in sorted(arm, key=lambda i: (-mets[i]["largest"], i))[:2]:
        take(i, "arm in the largest component (%d dofs), %s" % (mets[i]["largest"], "descent" if tags[i]["source"] == 1 else "closing"))
    # a contact capacity that ends inside the analytic contacts without cutting the candidate list (2 maxcon >= ncand, maxcon >= 16)
    room = [m["nanalytic"] - max(16, (m["ncand"] + 1) // 2) for m in mets]
    i = int(np.argmax(room))
    take(i, "%d analytic contacts, %d candidates" % (mets[i]["nanalytic"], mets[i]["ncand"]))
    with_contacts = [i for i in range(n) if mets[i]["ncon"] > 0 and tags[i]["source"] == 0]
    first = min(with_contacts, key=lambda i: (tags[i]["step"], tags[i]["seed"]))
    take(first, "earliest snapshot with contacts (%d)" % mets[first]["ncon"])
    # further big components, one per seed first, then by size
    big = sorted((i for i in range(n) if mets[i]["largest"] >= BIG_ISLAND), key=lambda i: (-mets[i]["blocks"], i))
    seen = {tags[i]["seed"] for i in chosen}
    for i in big:
        if len(chosen) >= N_SELECT:
            break
        if tags[i]["seed"] not in seen:
            take(i, "component of %d dofs (block sum %d)" % (mets[i]["largest"], mets[i]["blocks"]))
            seen.add(tags[i]["seed"])
    for i in big:
        if len(chosen) >= N_SELECT:
            break
        take(i, "component of %d dofs (block sum %d)" % (mets[i]["largest"], mets[i]["blocks"]))
    for i in sorted(range(n), key=lambda i: (-mets[i]["ncomp"], i)):
        if len(chosen) >= N_SELECT:
            break
        take(i, "%d components" % mets[i]["ncomp"])
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
    with Pool(min(len(SEEDS) + 1, os.cpu_count() or 1), maxtasksperchild=1) as pool:
        runs = pool.map(settle_run, list(SEEDS)) + pool.map(descent_run, [0])
        items = [it for r in runs for it in r]
        res = {}
        for so in (None, fast):
            out = pool.map(measure_all, [(items[c::8], so) for c in range(8)], chunksize=1)
            res[so] = [out[i % 8][i // 8] for i in range(len(items))]
    # a state whose forward() moves by more than a tenth of the tests' tolerances between two oracle builds is rounding-sensitive
    # (e.g. an MPR contact normal near an edge): the engine could not be held to the oracle on it
    ok = [robust(res[None][i], res[fast][i]) for i in range(len(items))]
    print("%d snapshots measured, %d rounding-sensitive ones dropped; no uncoupled tree has more than %d contacts (the group path "
          "takes 15)" % (len(items), ok.count(False), max(r[0]["uncoupled_tree_max_contacts"] for r in res[None])))
    items = [it for it, k in zip(items, ok) if k]
    mets = [r[0] for r, k in zip(res[None], ok) if k]
    tags = [t for t, _, _ in items]
    chosen, why = select(tags, mets)
    print("block sum above %d doubles: %d snapshots" % (HCAP_DEFAULT, sum(m["blocks"] > HCAP_DEFAULT for m in mets)))
    for i in chosen:
        t, m = tags[i], mets[i]
        print("%-8s seed %d step %4d: ncon %3d  components %2d  largest %3d dofs  block sum %4d  -- %s" % (
            ["settle", "descent", "closing"][t["source"]], t["seed"], t["step"], m["ncon"], m["ncomp"], m["largest"], m["blocks"], "; ".join(why[i])))
    arrays = {"qpos": np.array([items[i][1] for i in chosen]), "qvel": np.array([items[i][2] for i in chosen])}
    for k in ("source", "seed", "step"):
        arrays[k] = np.array([tags[i][k] for i in chosen], np.int32)
    for k in mets[0]:
        arrays[k] = np.array([mets[i][k] for i in chosen], np.int32)
    save_npz(OUT, arrays)


if __name__ == "__main__":
    main()
