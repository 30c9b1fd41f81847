"""Scene A1 (BASELINE configs 3 and 4: the 6-object scene with every object a 4 cm cube) against the fp64 oracle.

Fixture: tests/golden/scene_a1.npz (tests/golden/make_scene_a1_golden.py).  Two equal cubes that meet axis-aligned are an exact SAT tie
between their face axes (the strict `>` of col_box_box makes box 1 the reference), their parallel edge axes are skipped by the 1e-6
guard, and the reference-face clipping of two equal squares puts incident vertices exactly on the clip lines (kept by `da <= 0`).
Resets make cubes fall onto cubes (75 of the first 200 seeds); the settled scene holds 21-28 contacts, a grasp attempt up to 30, against
the warp-per-env build's 32-contact list.  Covered here:
  * one forward() of every stored state (reset snapshots and hand-built states): contacts (analytic 1e-9, MPR 1e-7), qacc and
    qfrc_constraint (1e-6 x scale), status and Newton iterations; a rounding-decided state may give one of the probe's other lists;
  * 60 sub-steps from every settle snapshot;
  * BatchedGraspEnv(200, "A1").reset() against the oracle's reset + stay(1000) of the same seeds;
  * every attempt record scattered over a 4096-env engine, and the episodes replayed attempt by attempt;
  * the contact list's headroom (status bit 0) and its behaviour at capacity;
  * top_down 200 x 200 images of the states, pixel for pixel.
"""
import os

import numpy as np
import pytest

from tests.common import contact_is_analytic

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAXCON = 32
TAGS = ["stack aligned", "stack offset x", "stack offset xy", "side by side", "stack rotated 1e-9", "bin wall stack", "held above cube"]
KIND_RESET, KIND_FIRST, KIND_TUMBLE, KIND_REST, KIND_BUILT = range(5)
CUBES = [30, 31, 32, 33, 34, 35]  # geom ids of the six cubes (box_1-3, ball_1-3 in scene A)
CUBE_QPOS = np.concatenate([np.arange(8 + 7 * i, 15 + 7 * i) for i in range(6)])
TABLE = 0.91


@pytest.fixture(scope="module")
def scene_a1():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    arrays, names = load_scene("A1")
    return load_scene_blob("A1"), arrays, names


@pytest.fixture(scope="module")
def fix():
    d = np.load(os.path.join(GOLD, "scene_a1.npz"))
    return {k: d[k] for k in d.files}


def _engine(blob, n, **env):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        return BatchedEngine(blob, n, 0)
    finally:
        for k in env:
            del os.environ[k]


def _oracle(blob, maxcon=MAXCON):
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(blob)
    o.set_maxcon(maxcon)
    return o


def _geom(o, g):
    return o.field("gpos").reshape(-1, 3)[g], o.field("gmat").reshape(-1, 3, 3)[g]


def _face_separations(o, g1, g2, h=0.02):
    """col_box_box's SAT separations along the face axes of box g1 (i) and of box g2 (j), in its order of operations"""
    (c1, R1), (c2, R2) = _geom(o, g1), _geom(o, g2)
    d = c2 - c1
    s1 = [abs(d[0] * R1[0, i] + d[1] * R1[1, i] + d[2] * R1[2, i]) - (h + h * abs(R1[:, i] @ R2[:, 0]) + h * abs(R1[:, i] @ R2[:, 1])
          + h * abs(R1[:, i] @ R2[:, 2])) for i in range(3)]
    s2 = [abs(d[0] * R2[0, j] + d[1] * R2[1, j] + d[2] * R2[2, j]) - (h + h * abs(R1[:, 0] @ R2[:, j]) + h * abs(R1[:, 1] @ R2[:, j])
          + h * abs(R1[:, 2] @ R2[:, j])) for j in range(3)]
    return s1, s2


def _cube_pair(o, g1=30, g2=31):
    bb = o.boxbox()
    row = bb[(bb[:, 0] == g1) & (bb[:, 1] == g2)]
    assert len(row) == 1, (g1, g2, bb)
    return row[0]


def _check_branch(tag, o):
    """the col_box_box branch a hand-built state is made for, on the oracle's geom frames (box_1 = geom 30 below, box_2 = 31)"""
    (c1, R1), (c2, R2) = _geom(o, 30), _geom(o, 31)
    rec = _cube_pair(o)  # geom1, geom2, outcome, reference, best axis, ties, guarded edge axes, on-line vertices, contacts
    s1, s2 = _face_separations(o, 30, 31)
    if tag in ("stack aligned", "stack offset x", "stack offset xy", "bin wall stack", "side by side"):
        assert np.array_equal(R1, np.eye(3)) and np.array_equal(R2, np.eye(3)), tag
        k = 1 if tag == "side by side" else 2  # the axis the cubes touch along
        # the two boxes' face axes along k tie bit for bit and are the largest: the strict `>` makes box_1 the reference
        assert s1[k] == s2[k] and s1[k] > max(s1[:k] + s1[k + 1:] + s2[:k] + s2[k + 1:]), (tag, s1, s2)
        assert tuple(rec[2:6]) == (1, 1, k, 2), (tag, rec)
        assert rec[6] == 0 and rec[8] == 4, (tag, rec)  # every cross product of two face axes is exactly 0 or 1 long
        if tag in ("stack aligned", "side by side"):
            # x faces coincide bit for bit (x = 0: x +- 0.02 is exact): the incident face's vertices lie on the clip lines x = +-h
            assert c1[0] == c2[0] == 0.0 and (c2[0] + 0.02) - c1[0] == 0.02 and (c2[0] - 0.02) - c1[0] == -0.02, tag
            assert rec[7] == 4, (tag, rec)
        elif tag == "stack offset x":
            assert c2[0] - c1[0] == 0.02 and c2[1] == c1[1], tag
        elif tag == "stack offset xy":
            assert c2[0] - c1[0] == 0.02 and abs(c2[1] - c1[1] - 0.02) < 1e-15, tag
        else:
            bin_wall = 0.6 - 0.2
            assert abs(c1[0] - 0.02 - bin_wall) < 1e-3 and abs(c2[0] - c1[0]) < 1e-15, tag  # against the bin's -x wall
    elif tag == "stack rotated 1e-9":
        assert np.array_equal(R1, np.eye(3))
        n = [np.linalg.norm(np.cross(R1[:, i], R2[:, j])) for i in range(3) for j in range(3)]
        assert sum(0 < v < 1e-6 for v in n) == 2 and min(v for v in n if v > 0) < 1e-8, n  # x-x and y-y: inside the guard
        assert s1[2] == s2[2] and rec[2] == 1 and rec[3] == 1 and rec[6] == 2 and rec[8] == 8, (s1, s2, rec)
    elif tag == "held above cube":
        assert c1[2] > TABLE + 0.05 and c2[2] < c1[2] and np.hypot(*(c1[:2] - c2[:2])) < 0.01
        pads = [g for g in range(30) if np.linalg.norm(_geom(o, g)[0] - c1) < 0.06]
        held = {int(c[14]) if int(c[13]) == 30 else int(c[13]) for c in o.contacts() if 30 in (int(c[13]), int(c[14]))} & set(pads)
        assert len(held) >= 2, ("not held between the fingers", held)
        assert rec[2] > 0 and rec[8] >= 1, rec
    else:
        raise AssertionError("untagged state " + tag)


def test_fixture_holds_a1_cases(fix):
    """cube-on-cube resets of every outcome kind, every tagged state, >= 64 single attempts with >= 40 rewarded, >= 4 episodes"""
    fell = fix["reset_fell"].astype(bool)
    up, tilt, on = fix["reset_up"], fix["reset_tilt"], fix["reset_on"]
    assert 0.25 < fell.mean() < 0.6, fell.mean()
    seeds = set(fix["state_seed"][fix["state_kind"] == KIND_REST].tolist())
    kinds = {"flip 90": False, "flip 180": False, "tilted": False, "stacked": False}
    for s in seeds:
        kinds["flip 90"] |= bool(((np.abs(up[s]) != 3) & (tilt[s] <= 5)).any())
        kinds["flip 180"] |= bool(((up[s] == -3) & (tilt[s] <= 5)).any())
        kinds["tilted"] |= bool((tilt[s] > 5).any())
        kinds["stacked"] |= bool(on[s].any())
    assert all(kinds.values()), kinds
    for k in (KIND_RESET, KIND_FIRST, KIND_TUMBLE, KIND_REST):
        assert (fix["state_kind"] == k).sum() >= 4, k
    assert sorted(fix["state_tag"][fix["state_kind"] == KIND_BUILT].tolist()) == list(range(len(TAGS)))
    assert len(fix["att_reward"]) >= 64 and fix["att_reward"].sum() >= 40 and fix["att_executed"].all()
    assert len(fix["episode_env"]) >= 4
    for e in fix["episode_env"]:
        assert list(fix["att_step"][fix["att_env"] == e]) == list(range(8)), e
    # the contact counts the generator measured: A1 settles at 21-28 contacts and an attempt peaks below the 32-contact list
    assert fix["reset_ncon"].max() <= MAXCON and fix["reset_peak"].max() <= MAXCON and fix["att_peak"].max() <= MAXCON
    assert fix["att_cap32_same"].all()


def test_a1_blob_is_the_transformed_scene(scene_a, scene_a1):
    """six boxes of half-size 0.02, each object body a uniform 4 cm cube at density 1000 (m = 0.064 kg, I = m (2h)^2 / 6), everything
    the transform does not reach equal to scene A's blob"""
    _, A, names = scene_a
    _, A1, names1 = scene_a1
    assert names == names1 and set(A) == set(A1)
    obj_geoms = [names["geom"].index(g) for g in ("box_1", "box_2", "box_3", "ball_1", "ball_2", "ball_3")]
    assert obj_geoms == CUBES
    gsize, gtype = np.asarray(A1["geom_size"]).reshape(-1, 3), np.ravel(A1["geom_type"])
    assert (gtype[CUBES] == 6).all() and (gsize[CUBES] == 0.02).all()
    obj_bodies = sorted({int(np.ravel(A1["geom_bodyid"])[g]) for g in CUBES})
    assert obj_bodies == list(range(18, 24))
    m = 1000.0 * 0.04 ** 3
    I = m * 0.04 ** 2 / 6
    mass, inertia = np.ravel(A1["body_mass"]), np.asarray(A1["body_inertia"]).reshape(len(np.ravel(A1["body_mass"])), -1)
    assert np.abs(mass[obj_bodies] - m).max() < 1e-12
    assert np.abs(inertia[obj_bodies, :3] - I).max() < 1e-12 and np.abs(inertia[obj_bodies, 3:]).max() < 1e-12
    other_b = [b for b in range(len(mass)) if b not in obj_bodies]
    other_g = [g for g in range(len(gtype)) if g not in CUBES]
    per_body = {"body_mass", "body_inertia", "body_invweight0"}
    per_geom = {"geom_type", "geom_size", "geom_rbound", "geom_obbhalf"}
    # derived from the objects' shapes and masses: the collision pair list and the inertia-dependent constants
    derived = {"pair_geom", "pair_rec", "pair_rsum", "tree_Minv", "dof_invweight0", "stat_meaninertia", "stat_extent"}
    for k in A:
        a, b = np.asarray(A[k]), np.asarray(A1[k])
        assert a.shape == b.shape, k
        if k in per_body:
            assert np.array_equal(a.reshape(len(mass), -1)[other_b], b.reshape(len(mass), -1)[other_b]), k
        elif k in per_geom:
            assert np.array_equal(a.reshape(len(gtype), -1)[other_g], b.reshape(len(gtype), -1)[other_g]), k
        elif k not in derived:
            assert np.array_equal(a, b), k
    # the arm's tree and its pairs are untouched
    tm, tm1 = np.asarray(A["tree_Minv"]), np.asarray(A1["tree_Minv"])
    assert np.array_equal(tm[0], tm1[0])
    pg, pg1 = np.asarray(A["pair_geom"]).reshape(-1, 2), np.asarray(A1["pair_geom"]).reshape(-1, 2)
    assert {tuple(p) for p in pg if not set(p) & set(CUBES)} == {tuple(p) for p in pg1 if not set(p) & set(CUBES)}


def test_tagged_states_reach_their_branches(scene_a1, fix):
    blob, A, _ = scene_a1
    o = _oracle(blob, 256)
    seen = set()
    for s in np.flatnonzero(fix["state_kind"] == KIND_BUILT):
        o.reset(fix["state_qpos"][s], fix["state_qvel"][s])
        o.forward()
        _check_branch(TAGS[fix["state_tag"][s]], o)
        seen.add(int(fix["state_tag"][s]))
    o.close()
    assert seen == set(range(len(TAGS)))


def test_fixture_is_what_the_oracle_produces_today(scene_a1, fix):
    """CPU: three stored attempts and three stored states re-run on the oracle, and one settled reset"""
    blob, A, _ = scene_a1
    from mujoco_rl_ur5_b200.batched_env import scene_a_reset_qpos

    o = _oracle(blob, 256)
    rew = np.flatnonzero(fix["att_reward"] == 1)
    for k in (int(rew[0]), int(np.flatnonzero(fix["att_reward"] == 0)[0]), len(fix["att_reward"]) - 1):
        o.reset(fix["att_q0"][k], fix["att_v0"][k])
        r, info = o.move_and_grasp(fix["att_coords"][k], int(fix["att_action"][k, 1]), 0.91)
        assert (r, info) == (int(fix["att_reward"][k]), fix["att_info"][k].tolist()), k
        assert np.abs(o.qpos[:8] - fix["att_arm_qpos"][k]).max() < 1e-9
    for s in (int(np.flatnonzero(fix["state_kind"] == KIND_FIRST)[0]), int(np.flatnonzero(fix["state_kind"] == KIND_REST)[-1]),
              int(np.flatnonzero(fix["state_kind"] == KIND_BUILT)[0])):
        o.reset(fix["state_qpos"][s], fix["state_qvel"][s])
        o.forward()
        assert o.ncon == fix["state_ncon"][s], s
    seed = int(np.flatnonzero(fix["reset_fell"])[0])
    o.reset(scene_a_reset_qpos(A, 20000 + seed))
    o.stay(1000)
    assert np.abs(o.qpos - fix["reset_qpos"][seed]).max() < 1e-12
    o.close()


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _alternatives(fix, s):
    """the contact lists a rounding-decided state may produce: (contacts, qacc, qfrc_constraint) of the probe's other lists"""
    out = []
    off = 0
    for k in range(len(fix["alt_state"])):
        n = int(fix["alt_ncon"][k])
        if fix["alt_state"][k] == s:
            out.append((fix["alt_contacts"][off:off + n], fix["alt_qacc"][k], fix["alt_qfrc_constraint"][k]))
        off += n
    return out


def _matches(A, gc, gq, gf, oc, oq, of):
    """None if the engine's forward() matches this oracle list within the GPU tolerances, else why not"""
    if gc.shape != oc.shape:
        return "ncon %d vs %d" % (len(gc), len(oc))
    if not np.array_equal(gc[:, 13:], oc[:, 13:]):
        return "geom ids / dims differ"
    if len(oc):
        tol = np.where(contact_is_analytic(A, oc), 1e-9, 1e-7)
        err = np.abs(gc[:, :13] - oc[:, :13]).max(axis=1)
        if not (err < tol).all():
            return "contact error %.3g (contact %d)" % (err.max(), int(np.argmax(err / tol)))
    for nm, g, r in (("qacc", gq, oq), ("qfrc_constraint", gf, of)):
        scale = max(1.0, float(np.abs(r).max()))
        if np.abs(g - r).max() > 1e-6 * scale:
            return "%s error %.3g (scale %.3g)" % (nm, float(np.abs(g - r).max()), scale)
    return None


@pytest.mark.gpu
def test_stage_parity_on_every_state(scene_a1, fix):
    """one forward() of every stored state: the oracle's contact list (or, for a rounding-decided state, one the probe recorded),
    qacc and qfrc_constraint, status 0 and the oracle's Newton iteration count"""
    blob, A, _ = scene_a1
    eng = _engine(blob, 1)
    o = _oracle(blob)
    bad, alt_used = [], 0
    try:
        assert eng.size(6) == MAXCON
        for s in range(len(fix["state_qpos"])):
            q, v = fix["state_qpos"][s], fix["state_qvel"][s]
            o.reset(q, v)
            o.forward()
            eng.set_state(q[None], v[None])
            g = {f: eng.debug_forward(0, f) for f in ("contact", "ncon", "qacc", "qfrc_constraint", "status", "niter")}
            gc = g["contact"].reshape(-1, 16)
            why = _matches(A, gc, g["qacc"], g["qfrc_constraint"], o.contacts(), o.field("qacc"), o.field("qfrc_constraint"))
            if why and fix["state_flag"][s]:
                for alt in _alternatives(fix, s):
                    if _matches(A, gc, g["qacc"], g["qfrc_constraint"], *alt) is None:
                        why, alt_used = None, alt_used + 1
                        break
            if why:
                bad.append((s, int(fix["state_kind"][s]), int(fix["state_tag"][s]), why))
            if int(g["status"][0]) != 0:
                bad.append((s, "status", int(g["status"][0])))
            if not fix["state_flag"][s] and abs(int(g["niter"][0]) - o.solver_iter) > (1 if o.ncon else 0):
                bad.append((s, "niter", int(g["niter"][0]), o.solver_iter))
    finally:
        eng.close()
        o.close()
    print("%d states, %d rounding-decided, %d matched an alternative list" % (len(fix["state_qpos"]), int(fix["state_flag"].sum()), alt_used))
    assert not bad, bad


@pytest.mark.gpu
def test_trajectory_parity_from_settle_snapshots(scene_a1, fix):
    """60 PID + sub-steps from every settle snapshot that is not rounding-decided, all in one batch: qpos within 1e-6 of the oracle"""
    blob, A, _ = scene_a1
    sel = np.flatnonzero(np.isin(fix["state_kind"], (KIND_RESET, KIND_FIRST, KIND_TUMBLE, KIND_REST)) & (fix["state_flag"] == 0))
    q, v = fix["state_qpos"][sel], fix["state_qvel"][sel]
    eng = _engine(blob, len(sel))
    try:
        eng.set_state(q, v)
        eng.move_group("All", None, 1e-9, 60)
        assert eng.run() == 0
        gq = eng.get_state()[0].cpu().numpy()
        st = eng.status().cpu().numpy()
    finally:
        eng.close()
    o = _oracle(blob)
    worst = 0.0
    for e, s in enumerate(sel):
        o.reset(q[e], v[e])
        o.move_group("All", None, 1e-9, 60)
        err = float(np.abs(gq[e] - o.qpos).max())
        worst = max(worst, err)
        assert err < 1e-6, (int(s), err)
        assert st[e] == 0, (int(s), int(st[e]))
    o.close()
    print("%d snapshots, worst |qpos - oracle| %.3g" % (len(sel), worst))


def _outcome(A, q):
    from tests.golden.make_scene_a1_golden import outcome

    up, _, on = outcome(A, q)
    return up, on


@pytest.mark.gpu
def test_reset_parity_through_the_facade(scene_a1, fix):
    """BatchedGraspEnv(200, "A1").reset() = the oracle's reset + stay(1000) of seeds 20000..20199: each cube's pose within 1e-6 where
    the oracle's two builds agree to 1e-8, else each cube's upward body axis and table-or-cube support as one of the two builds"""
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    blob, A, _ = scene_a1
    n = len(fix["reset_qpos"])
    env = BatchedGraspEnv(n, "A1", 0)
    try:
        env.reset()
        gq = env.engine.get_state()[0].cpu().numpy()
        st = env.engine.status().cpu().numpy()
    finally:
        env.close()
    bad, worst = [], 0.0
    for i in range(n):
        if fix["reset_robust"][i]:
            err = float(np.abs(gq[i][CUBE_QPOS] - fix["reset_qpos"][i][CUBE_QPOS]).max())
            worst = max(worst, err)
            if err > 1e-6:
                bad.append((i, "pose", err))
        else:
            up, on = _outcome(A, gq[i])
            if not any(np.array_equal(up, fix[u][i]) and np.array_equal(on, fix[c][i])
                       for u, c in (("reset_up", "reset_on"), ("reset_up_fast", "reset_on_fast"))):
                bad.append((i, "outcome", up.tolist(), fix["reset_up"][i].tolist()))
    print("%d resets (%d cube-on-cube falls, %d compared by pose), worst pose error %.3g, status bits seen %s" % (
        n, int(fix["reset_fell"].sum()), int(fix["reset_robust"].sum()), worst, sorted(set(st.tolist()))))
    assert (st == 0).all(), np.flatnonzero(st)
    assert not bad, bad


def _wave_boundaries(n):
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {0, 3, 4, 9, 10, n - 1}
    for per_sm in (8, 10):  # resident envs per SM of the warp-per-env build (ten: one CTA of ten warps or two of five)
        for w in (1, 2, 3):
            out |= {w * sms * per_sm - 1, w * sms * per_sm}
    return sorted(e for e in out if 0 <= e < n)


@pytest.mark.gpu
def test_attempts_at_the_bench_size(scene_a1, fix):
    """4096 envs, every attempt record scattered over them (rewarded records at env 0, 4095 and the CTA / wave boundaries), one
    BatchedGraspEnv.step: executed flag and reward bit-exact, the 12 phase counters exact, arm angles 1e-4, depth at the action
    pixel 1e-4 m, status 0, and every copy of a record bit-identical to the others"""
    import torch

    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    R, N = len(fix["att_reward"]), 4096
    which = np.arange(N) % R
    rew = np.flatnonzero(fix["att_reward"] == 1)
    for j, e in enumerate(_wave_boundaries(N)):
        which[e] = rew[(5 * j) % len(rew)]
    env = BatchedGraspEnv(N, "A1", 0)
    try:
        env.engine.set_state(fix["att_q0"][which], fix["att_v0"][which])
        env.current_observation = None
        actions = fix["att_action"][which].astype(np.int32)
        depth0 = env.get_observation()["depth"]
        dev = depth0.device
        d_at = depth0[torch.arange(N, device=dev), torch.as_tensor(actions[:, 0] // 200, device=dev).long(),
                      torch.as_tensor(actions[:, 0] % 200, device=dev).long()].cpu().numpy()
        _, reward, _, info = env.step(actions)
        executed = info["executed"].cpu().numpy().astype(bool)
        ginfo = env.engine.grasp_info().cpu().numpy()
        qpos = env.engine.get_state()[0].cpu().numpy()
        status = env.engine.status().cpu().numpy()
    finally:
        env.close()
    bad = []
    worst_d = float(np.abs(d_at - fix["att_depth"][which]).max())
    worst_q = float(np.abs(qpos[:, :8] - fix["att_arm_qpos"][which]).max())
    for e in np.flatnonzero((executed != fix["att_executed"][which].astype(bool)) | (reward != fix["att_reward"][which])
                            | (ginfo != fix["att_info"][which]).any(axis=1)
                            | (np.abs(qpos[:, :8] - fix["att_arm_qpos"][which]).max(axis=1) > 1e-4)):
        bad.append((int(e), int(which[e]), int(reward[e]), int(fix["att_reward"][which[e]]), ginfo[e].tolist(), fix["att_info"][which[e]].tolist()))
    for w in range(R):
        idx = np.flatnonzero(which == w)
        if not (qpos[idx] == qpos[idx[0]]).all():
            bad.append(("copies differ", w))
    print("A1 at %d envs: %d records, %d rewarded attempts expected, worst arm dq %.2e, worst depth diff %.2e, status bits %s, %d mismatches"
          % (N, R, int(fix["att_reward"][which].sum()), worst_q, worst_d, sorted(set(status.tolist())), len(bad)))
    assert worst_d < 1e-4
    assert (status == 0).all(), np.flatnonzero(status)[:10]
    assert not bad, bad[:10]


@pytest.mark.gpu
def test_episodes_attempt_by_attempt(scene_a1, fix):
    """the stored episodes (8 consecutive attempts from one reset, cubes piling up in the drop bin), re-synchronised to the oracle's
    state before every attempt: 0 mismatches in reward and phase counters, arm within 1e-4, status bit 0 never set"""
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    envs = fix["episode_env"]
    env = BatchedGraspEnv(len(envs), "A1", 0)
    mism, statuses = [], set()
    try:
        for k in range(8):
            rec = np.array([int(np.flatnonzero((fix["att_env"] == e) & (fix["att_step"] == k))[0]) for e in envs])
            env.engine.set_state(fix["att_q0"][rec], fix["att_v0"][rec])
            env.current_observation = None
            _, reward, _, _ = env.step(fix["att_action"][rec].astype(np.int32))
            ginfo = env.engine.grasp_info().cpu().numpy()
            qpos = env.engine.get_state()[0].cpu().numpy()
            statuses |= set(env.engine.status().cpu().numpy().tolist())
            for j, r in enumerate(rec):
                if int(reward[j]) != fix["att_reward"][r] or ginfo[j].tolist() != fix["att_info"][r].tolist() or \
                        np.abs(qpos[j, :8] - fix["att_arm_qpos"][r]).max() > 1e-4:
                    mism.append((int(envs[j]), k, int(reward[j]), int(fix["att_reward"][r])))
    finally:
        env.close()
    print("episodes %s: %d attempts, %d rewarded, status bits %s" % (envs.tolist(), 8 * len(envs),
                                                                     int(sum(fix["att_reward"][np.isin(fix["att_env"], envs)])), sorted(statuses)))
    assert not any(s & 1 for s in statuses) and statuses <= {0}, statuses
    assert not mism, mism


@pytest.mark.gpu
def test_no_contact_overflow_at_4096_envs_config_3(scene_a1):
    """the config-3 workload: 4096 A1 envs reset, then two steps of random table actions; no env sets status bit 0 (the 32-contact
    list overflowed) or any other bit"""
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    N = 4096
    rng = np.random.RandomState(0)
    env = BatchedGraspEnv(N, "A1", 0)
    seen = []
    try:
        env.reset()
        seen.append(env.engine.status().cpu().numpy())
        for _ in range(2):
            px, py = rng.randint(40, 160, N), rng.randint(60, 140, N)
            env.step(np.stack([py * 200 + px, rng.randint(0, 6, N)], axis=1))
            seen.append(env.engine.status().cpu().numpy())
    finally:
        env.close()
    for k, st in enumerate(seen):
        print("after %s: %d envs with bit 0, %d flagged" % (["reset", "step 1", "step 2"][k], int((st & 1).sum()), int((st != 0).sum())))
    assert all((st == 0).all() for st in seen)


@pytest.mark.gpu
def test_contact_list_at_capacity(scene_a1, fix):
    """GE_MAXCON = ncon, ncon - 1 and a cut inside a cube-cube pair's manifold, on the states with the most contacts: the engine's
    list is the oracle's first maxcon contacts under set_maxcon, status bit 0 iff more were found, qacc the capped oracle's"""
    blob, A, _ = scene_a1
    cands = np.argsort(-fix["state_ncon"], kind="stable")[:3].tolist()
    cands.append(int(np.flatnonzero((fix["state_kind"] == KIND_BUILT) & (fix["state_tag"] == TAGS.index("stack rotated 1e-9")))[0]))
    o = _oracle(blob, 256)
    checked, inside = 0, 0
    try:
        for s in cands:
            q, v = fix["state_qpos"][s], fix["state_qvel"][s]
            o.set_maxcon(256)
            o.reset(q, v)
            o.forward()
            total, ncand, oc = o.ncon, o.ncand, o.contacts()
            caps = [total, total - 1]
            for start in range(total):  # the first cube-cube manifold of two or more points: cut after its first point
                g1, g2 = int(oc[start, 13]), int(oc[start, 14])
                if g1 in CUBES and g2 in CUBES and start + 1 < total and oc[start + 1, 13] == g1 and oc[start + 1, 14] == g2:
                    caps.append(start + 1)
                    inside += 1
                    break
            for cap in dict.fromkeys(caps):
                if cap < 16 or 2 * cap < ncand:
                    continue
                eng = _engine(blob, 1, GE_MAXCON=cap)
                try:
                    assert eng.size(6) == cap
                    eng.set_state(q[None], v[None])
                    g = {f: eng.debug_forward(0, f) for f in ("contact", "ncon", "status", "qacc", "qfrc_constraint")}
                finally:
                    eng.close()
                o.set_maxcon(cap)
                o.reset(q, v)
                o.forward()
                st = int(g["status"][0])
                assert o.con_overflow == int(total > cap)
                assert int(g["ncon"][0]) == min(total, cap) == o.ncon, (s, cap, int(g["ncon"][0]), total)
                assert (st & 1) == int(total > cap) and not st & ~1, (s, cap, st)
                why = _matches(A, g["contact"].reshape(-1, 16), g["qacc"], g["qfrc_constraint"], o.contacts(), o.field("qacc"),
                               o.field("qfrc_constraint"))
                assert why is None, (s, cap, why)
                checked += 1
    finally:
        o.close()
    print("capacity cases checked: %d (%d cuts inside a cube-cube manifold)" % (checked, inside))
    assert checked >= 6 and inside >= 1


@pytest.mark.gpu
def test_render_top_down(scene_a1, fix):
    """top_down 200 x 200 images of every stored state and of the attempt records' start states: every pixel equals the oracle's
    except where its render probe flags rounding (tests/test_render_edges_gpu.py's rule)"""
    from tests.test_render_edges_gpu import EPS_M, EPS_PX

    blob, A, _ = scene_a1
    cam = int(np.ravel(A["cam_top_down"])[0])
    states = list(fix["state_qpos"]) + list(fix["att_q0"][::8])
    eng = _engine(blob, len(states))
    try:
        eng.set_state(np.stack(states))
        rgb, depth = eng.render(cam, 200, 200)
        rgb, depth = rgb.cpu().numpy(), depth.cpu().numpy()
    finally:
        eng.close()
    o = _oracle(blob, 256)
    failures, mism, flagged = [], 0, 0
    for k, q in enumerate(states):
        o.reset(q)
        orgb, odepth = o.render(cam, 200, 200)
        diff = (depth[k].view(np.uint32) != odepth.view(np.uint32)) | (rgb[k] != orgb).any(axis=2)
        idx = np.flatnonzero(diff)
        mism += len(idx)
        if len(idx):
            fl = o.render_probe(cam, 200, 200, idx, EPS_PX, EPS_M)[1]
            flagged += int((fl != 0).sum())
            if (fl == 0).any():
                failures.append((k, int((fl == 0).sum()), [(int(i // 200), int(i % 200)) for i in idx[fl == 0][:4]]))
    o.close()
    print("%d images: %d mismatching pixels, %d of them flagged" % (len(states), mism, flagged))
    assert not failures, failures
