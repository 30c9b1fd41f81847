"""Joint-limit rows, the 16 simple-row slots and the degenerate branches of the narrow phase, in both builds, against the fp64 oracle.

Fixture: tests/golden/limits_contacts.npz (tests/golden/make_limits_contacts_golden.py), constructed states each tagged with the branch
it targets.  Until this file, no tested state built a joint-limit row (efc_type 1), so the limit loop of stage_constraints (its ordered
compaction over 32 / 128 lanes, the lower / upper sign, the aref with the margin), the active set of a limit row in nt_update and the
simple-row slots 1..15 had never been compared with the oracle; nor had the branches where a contact function divides by something near
zero or picks between ties.  Covered here:
  * CPU pins: each state reaches its tagged branch (plain-Python predicates in the body frame, the oracle's rows split into equality,
    limit and contact rows), the oracle's limit rows equal a plain restatement of make_constraint's rule, its simple-row cap, and that
    both trajectories really build limit rows;
  * stage parity in the warp-per-env build (scene A) and the CTA-per-env build (scene B): nsr, contacts, qacc, qfrc_constraint,
    status and Newton iterations;
  * the capacity: 16 simple rows fit (status 0), 17 set GE_STATUS_ROW_OVERFLOW (and not CONTACT_OVERFLOW) and solve what the oracle
    solves with set_maxsr(16);
  * an open-loop run into shoulder_lift's upper limit (step_open_loop) and a move_group beyond it (k_run) against the oracle;
  * 30 envs, ten to a CTA, limit-heavy states among ordinary ones: each bit-identical to the same state run alone.
"""
import os
import re

import numpy as np
import pytest

from tests.common import contact_is_analytic

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "limits_contacts.npz")
EDGES_A = os.path.join(HERE, "golden", "scene_a_edges.npz")
MAXSR = 16
ROW_OVERFLOW, CONTACT_OVERFLOW = 8, 1
WIDTH, MID = 0.001, 0.5  # jnt_solimp[2:4] of both scenes


@pytest.fixture(scope="module")
def fix():
    d = np.load(FIXTURE)
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


def _states(fix, scene):
    s = "_" + scene.lower()
    return [(str(t), q, v) for t, q, v in zip(fix["tag" + s], fix["qpos" + s], fix["qvel" + s])]


def _forward(blob, q, v, maxsr=-1):
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(blob)
    o.set_maxsr(maxsr)
    o.reset(q, v)
    o.forward()
    return o


def limit_rows(A, q):
    """make_constraint's limit rule, restated: every limited joint in joint order, lower side first, a row where the distance to the
    range end is below the margin; (joint, dof, sign of the Jacobian entry, distance)"""
    out = []
    rng = np.asarray(A["jnt_range"]).reshape(-1, 2)
    lim, mg = np.asarray(A["jnt_limited"]).ravel(), np.asarray(A["jnt_margin"]).ravel()
    qa, da = np.asarray(A["jnt_qposadr"]).ravel(), np.asarray(A["jnt_dofadr"]).ravel()
    for j in range(len(lim)):
        if lim[j]:
            for side, dist in ((0, q[qa[j]] - rng[j, 0]), (1, rng[j, 1] - q[qa[j]])):
                if dist < mg[j]:
                    out.append((j, int(da[j]), 1.0 if side == 0 else -1.0, dist))
    return out


def _geom(o, g):
    return o.field("gpos").reshape(-1, 3)[g], o.field("gmat").reshape(-1, 3, 3)[g]


def _contact_predicate(tag, o, A):
    """the narrow-phase branch a contact state is built for, checked on the oracle's geom frames"""
    size = np.asarray(A["geom_size"]).reshape(-1, 3)
    if tag.startswith("sphere centre inside box"):
        (cs, _), (cb, Rb) = _geom(o, 33), _geom(o, 32)  # ball_1 in box_3
        p = Rb.T @ (cs - cb)
        h = size[32]
        assert (np.abs(p) <= h).all()
        slack = h - np.abs(p)
        k = int(tag[-1])
        assert slack.argmin() == k and np.sort(slack)[1] > slack[k] + 1e-3, (tag, slack)
    elif tag == "sphere-sphere coincident centres":
        assert np.linalg.norm(_geom(o, 33)[0] - _geom(o, 34)[0]) < 1e-15
    elif tag == "aligned box-box stack":
        (c1, R1), (c3, R3) = _geom(o, 30), _geom(o, 32)
        assert np.array_equal(R1, np.eye(3)) and np.array_equal(R3, np.eye(3))
        # col_box_box's SAT separations along the face axes of box_1 (i) and box_3 (j), in its order of operations: along z they tie
        # bit for bit and are the largest, so the strict `>` decides which box is the reference
        d, h1, h2 = c3 - c1, size[30], size[32]
        s1 = [abs(d @ R1[:, i]) - (h1[i] + h2[0] * abs(R1[:, i] @ R3[:, 0]) + h2[1] * abs(R1[:, i] @ R3[:, 1]) + h2[2] * abs(R1[:, i] @ R3[:, 2]))
              for i in range(3)]
        s2 = [abs(d @ R3[:, j]) - (h2[j] + h1[0] * abs(R1[:, 0] @ R3[:, j]) + h1[1] * abs(R1[:, 1] @ R3[:, j]) + h1[2] * abs(R1[:, 2] @ R3[:, j]))
              for j in range(3)]
        assert s1[2] == s2[2] and s1[2] > max(s1[:2] + s2[:2]), (s1, s2)
    elif tag == "capsule-capsule parallel":
        a1, a2 = _geom(o, 60)[1][:, 2], _geom(o, 61)[1][:, 2]
        assert 1 - np.dot(a1, a2) ** 2 < 1e-10
    elif tag == "capsule-capsule crossing axes":
        (p1, R1), (p2, R2) = _geom(o, 60), _geom(o, 62)
        n = np.cross(R1[:, 2], R2[:, 2])
        assert abs(np.dot(p2 - p1, n)) < 1e-12 and np.linalg.norm(n) > 0.99  # the axes intersect
    elif tag.startswith("sphere centre inside cylinder"):
        (cs, _), (cc, Rc) = _geom(o, 30), _geom(o, 50)
        l = Rc.T @ (cs - cc)
        dr, dz = np.hypot(l[0], l[1]) - size[50, 0], abs(l[2]) - size[50, 1]
        assert dr <= 0 and dz <= 0 and ((dr > dz) == tag.endswith("radial")), (tag, dr, dz)
    elif tag == "sphere centre on capsule axis":
        (cs, _), (cc, Rc) = _geom(o, 31), _geom(o, 60)
        t = np.dot(cs - cc, Rc[:, 2])
        assert abs(t) < size[60, 1] and np.linalg.norm(cc + t * Rc[:, 2] - cs) < 1e-12
    elif tag == "upright cylinder on the floor":
        ax = _geom(o, 51)[1][:, 2]
        assert np.linalg.norm(ax - [0, 0, 1]) < 1e-12  # the rim direction vanishes
    elif tag == "capsule coaxial on upright cylinder":
        (pc, Rc), (pk, Rk) = _geom(o, 50), _geom(o, 63)
        assert np.array_equal(Rc[:, 2], [0, 0, 1]) and np.array_equal(Rk[:, 2], [0, 0, 1]) and np.array_equal(pc[:2], pk[:2])
    else:
        raise AssertionError("untagged contact state " + tag)


def test_states_reach_their_branches(scene_a, scene_b, fix):
    """each state reaches its tagged branch; the oracle's limit rows are the restated rule's, with |pos| / width in the tagged
    impedance band; the trajectories' start states and the contact states build no limit row"""
    seen = set()
    for scene, (blob, A, _) in (("A", scene_a), ("B", scene_b)):
        nv = int(np.asarray(A["nv"]).ravel()[0])
        for tag, q, v in _states(fix, scene):
            o = _forward(blob, q, v)
            ne, nl, nc = o.efc_split
            assert ne == 1 and o.nefc == ne + nl + nc
            assert nc == sum(1 if c[15] == 1 else 2 * (int(c[15]) - 1) for c in o.contacts())
            rows = limit_rows(A, q)
            assert nl == len(rows), (tag, nl, len(rows))
            J = o.field("efc_J").reshape(-1, nv)[ne:ne + nl] if nl else np.zeros((0, nv))
            pos = o.field("efc_pos")[ne:ne + nl]
            for r, (j, d, sgn, dist) in enumerate(rows):
                assert J[r, d] == sgn and np.count_nonzero(J[r]) == 1 and pos[r] == dist, (tag, r, j)
            if scene == "A" and tag.startswith(("open loop", "move_group")):
                assert nl == 0
            elif tag.startswith("capacity"):
                assert nl == int(tag.split()[1])
                seen.add(("A", "capacity", ne + nl))
            elif "limit" in tag:
                assert nl > 0, tag
                if " d" in tag:  # one limit, at a tagged depth: x = |dist| / width in the tagged impedance band
                    depth = float(tag.split(" d")[1].split()[0])
                    x = np.abs(pos) / WIDTH
                    assert np.allclose(x, depth / WIDTH)
                    band = 0 if depth / WIDTH <= MID else (1 if depth / WIDTH < 1 else 2)
                    seen.add((scene, "impedance", band))
                    j = rows[0][0]
                    seen.add((scene, "joint", j, "upper" if rows[0][2] < 0 else "lower"))
                if nl:
                    f = o.field("efc_force")[ne:ne + nl]
                    seen.update((scene, "active" if fr != 0 else "inactive") for fr in f)
            else:
                assert nl == 0 and o.ncon >= 1
                _contact_predicate(tag, o, A)
                seen.add((scene, tag))
            o.close()
    for band in range(3):
        assert ("A", "impedance", band) in seen and ("B", "impedance", band) in seen
    assert {("A", "active"), ("A", "inactive"), ("B", "active"), ("B", "inactive")} <= seen
    assert {("A", "capacity", n) for n in (15, 16, 17)} <= seen
    assert ("A", "joint", 1, "upper") in seen and ("A", "joint", 3, "lower") in seen and ("A", "joint", 6, "upper") in seen
    assert sum(1 for s in seen if s[0] == "A" and s[1] == "joint" and s[2] >= 8) >= 3  # object slides: x, y and z
    assert len([s for s in seen if len(s) == 2 and s[1] not in ("active", "inactive")]) == 12


def test_oracle_simple_row_cap(scene_a, fix):
    """set_maxsr(16) keeps the equality row and the first 15 limit rows in joint order: nothing changes up to 16 rows, the 17th is
    dropped (sr_overflow) and the solve changes with it; no contact is lost"""
    blob, A, _ = scene_a
    for tag, q, v in _states(fix, "A"):
        if not tag.startswith("capacity"):
            continue
        full, cap = _forward(blob, q, v), _forward(blob, q, v, MAXSR)
        ne, nl, nc = full.efc_split
        over = ne + nl > MAXSR
        assert cap.efc_split == (ne, min(nl, MAXSR - ne), nc) and cap.sr_overflow == int(over) and full.sr_overflow == 0
        assert np.array_equal(cap.field("efc_pos")[:MAXSR], full.field("efc_pos")[:MAXSR])
        assert np.array_equal(cap.contacts(), full.contacts())
        assert np.array_equal(cap.field("qacc"), full.field("qacc")) != over, tag
        full.close()
        cap.close()


def _row_states_open_loop(blob, fix, q, v):
    """per sub-step of the open-loop run: 0 no limit row, 1 shoulder_lift's row inactive, 2 active"""
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(blob)
    o.reset(q, v)
    seq = []
    for ctrl, n in zip(fix["open_loop_ctrl"], fix["open_loop_steps"]):
        o.ctrl[:] = ctrl
        for _ in range(int(n)):
            o.forward()
            ne, nl, _ = o.efc_split
            seq.append(0 if nl == 0 else 1 + int(o.field("efc_force")[ne] != 0))
            o.step()
    o.close()
    return "".join(map(str, seq))


def _tagged(fix, scene, prefix):
    return next((q, v) for t, q, v in _states(fix, scene) if t.startswith(prefix))


def test_trajectories_build_limit_rows(scene_a, fix):
    """the open-loop run drives shoulder_lift into its upper limit and its row goes active -> inactive -> active; the move_group beyond
    that limit ends in max-steps, and the oracle builds limit rows on its way"""
    blob, A, _ = scene_a
    seq = _row_states_open_loop(blob, fix, *_tagged(fix, "A", "open loop"))
    print("open loop, shoulder_lift's row per sub-step:", seq)
    assert re.fullmatch("0+2+1+2+", seq), seq
    from oracle.oracle_py import OracleEnv

    q, v = _tagged(fix, "A", "move_group")
    o = OracleEnv(blob)
    o.reset(q, v)
    nls = []
    for _ in range(int(fix["beyond_steps"].item()) // 10):  # the same movement in chunks, to look at the rows on the way
        o.move_group("All", fix["beyond_target"], 1e-7, 10)
        o.forward()
        nls.append(o.efc_split[1])
    o.reset(q, v)
    assert o.move_group("All", fix["beyond_target"], 1e-7, int(fix["beyond_steps"].item())) == (2, int(fix["beyond_steps"].item()) + 1)
    o.close()
    print("move_group beyond the limit, limit rows every 10 sub-steps:", nls)
    assert fix["beyond_target"][1] > np.asarray(A["jnt_range"]).reshape(-1, 2)[1, 1] and max(nls) > 0


def _check(A, g, o, what):
    """one engine forward() against the oracle's: rows, contacts, qacc / qfrc_constraint, iterations"""
    ne, nl, _ = o.efc_split
    assert int(g["nsr"][0]) == ne + nl, (what, int(g["nsr"][0]), ne + nl)
    oc, gc = o.contacts(), g["contact"].reshape(-1, 16)
    assert int(g["ncon"][0]) == o.ncon and gc.shape == oc.shape, (what, int(g["ncon"][0]), o.ncon)
    assert np.array_equal(gc[:, 13:], oc[:, 13:]), (what, "contact geom ids / dims differ")
    if len(oc):
        tol = np.where(contact_is_analytic(A, oc), 1e-9, 1e-7)
        err = np.abs(gc[:, :13] - oc[:, :13]).max(axis=1)
        assert (err < tol).all(), (what, err.max())
    for f in ("qacc", "qfrc_constraint"):
        r = o.field(f)
        scale = max(1.0, float(np.abs(r).max()))
        err = float(np.abs(g[f] - r).max())
        assert err <= 1e-7 * scale, (what, f, err, scale)
    # Newton iterations: exact without contacts (the simple rows are the oracle's rows, term for term); with contacts within one, since
    # the matrix-free contact rows sum in another order and the last stop test compares a cost decrease with the tolerance (the
    # oracle's own -ffp-contract=fast build takes one iteration more than its checker build on an arm state with 14 contacts)
    assert abs(int(g["niter"][0]) - o.solver_iter) <= (1 if o.ncon else 0), (what, int(g["niter"][0]), o.solver_iter)


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["A", "B"])
def test_stage_parity(scene_a, scene_b, fix, scene):
    """every state, one forward(): nsr = the oracle's equality + limit rows, contacts (analytic 1e-9, MPR 1e-7, ids and dims exact),
    qacc and qfrc_constraint within 1e-7 relative, status and Newton iterations (within one when there are contacts); 17 simple rows are checked against the oracle capped
    at 16 and must set ROW_OVERFLOW, never CONTACT_OVERFLOW"""
    blob, A, _ = scene_a if scene == "A" else scene_b
    eng = _engine(blob, 1)
    fields = ("qacc", "qfrc_constraint", "contact", "ncon", "niter", "nsr", "status")
    report = []
    try:
        assert eng.size(9) == (0 if scene == "A" else 1) and (scene == "B" or eng.size(8) == 10)
        for tag, q, v in _states(fix, scene):
            full = _forward(blob, q, v)
            ne, nl, _ = full.efc_split
            over = ne + nl > MAXSR
            o = _forward(blob, q, v, MAXSR) if over else full
            eng.set_state(q[None], v[None])
            g = {f: eng.debug_forward(0, f) for f in fields}
            st = int(g["status"][0])
            assert st == (ROW_OVERFLOW if over else 0), (tag, st)
            _check(A, g, o, tag)
            if over:
                assert int(g["nsr"][0]) == MAXSR and o.sr_overflow
                assert not np.array_equal(full.field("qacc"), o.field("qacc"))  # the dropped row mattered
            report.append((tag, int(g["nsr"][0]), int(g["ncon"][0]), int(g["niter"][0]), st))
            if o is not full:
                o.close()
            full.close()
    finally:
        eng.close()
    print("state, nsr, ncon, niter, status:", report)
    assert len(report) == len(fix["tag_" + scene.lower()])


@pytest.mark.gpu
def test_trajectories(scene_a, fix):
    """the open-loop run into shoulder_lift's upper limit through step_open_loop (each control phase in two calls) and the move_group
    beyond it through k_run: qpos within 1e-6 and qvel within 1e-4 of the oracle, result and step count equal"""
    from oracle.oracle_py import OracleEnv

    blob, A, _ = scene_a
    eng = _engine(blob, 1)
    o = OracleEnv(blob)
    try:
        q, v = _tagged(fix, "A", "open loop")
        eng.set_state(q[None], v[None])
        o.reset(q, v)
        for ctrl, n in zip(fix["open_loop_ctrl"], fix["open_loop_steps"]):
            eng.set_ctrl(ctrl[None])
            for k in ((1, int(n) - 1) if n > 1 else (1,)):
                eng.step_open_loop(k)
            o.ctrl[:] = ctrl
            o.step(int(n))
        gq, gv = (x.cpu().numpy()[0] for x in eng.get_state())
        assert np.abs(gq - o.qpos).max() < 1e-6 and np.abs(gv - o.qvel).max() < 1e-4, (np.abs(gq - o.qpos).max(), np.abs(gv - o.qvel).max())
        assert int(eng.status()[0]) == 0
        q, v = _tagged(fix, "A", "move_group")
        m = int(fix["beyond_steps"].item())
        eng.set_state(q[None], v[None])
        eng.move_group("All", fix["beyond_target"][None], 1e-7, m)
        assert eng.run() == 0
        res, steps, _, _ = eng.results()
        o.reset(q, v)
        r, s = o.move_group("All", fix["beyond_target"], 1e-7, m)
        gq, gv = (x.cpu().numpy()[0] for x in eng.get_state())
        assert (int(res[0]), int(steps[0])) == (r, s) == (2, m + 1)
        assert np.abs(gq - o.qpos).max() < 1e-6 and np.abs(gv - o.qvel).max() < 1e-4, (np.abs(gq - o.qpos).max(), np.abs(gv - o.qvel).max())
    finally:
        eng.close()
        o.close()


def _targets(q):
    return q[:, :7] + np.array([0.02, -0.02, 0.02, 0.01, 0.01, 0.05, 0.0])


@pytest.mark.gpu
def test_limit_rows_beside_other_envs(scene_a, fix):
    """30 envs through one k_run, ten to a CTA: in every CTA the two states of 15 and 16 simple rows (slots 1..15 live in the
    lifetime-aliased scratch region of the warp-per-env build, over cinert and the RNE / CRB temporaries), four single-limit states and
    four of the capacity-edge fixture's states; 60 PID + sub-steps, each env's qpos, qvel and status bit-identical to the same state run
    alone"""
    blob, A, _ = scene_a
    nsr = {}
    limit = []
    for t, q, v in _states(fix, "A"):
        o = _forward(blob, q, v)
        ne, nl, _ = o.efc_split
        o.close()
        if nl and ne + nl <= MAXSR:
            nsr[id(q)] = ne + nl
            limit.append((q, v))
    heavy = sorted(limit, key=lambda s: -nsr[id(s[0])])[:2]
    single_rows = [s for s in limit if nsr[id(s[0])] <= 3]
    edges = np.load(EDGES_A)
    theirs = list(zip(edges["qpos"], edges["qvel"]))
    states = []
    for c in range(3):
        mine = heavy + single_rows[4 * c:4 * c + 4]
        other = [theirs[(4 * c + k) % len(theirs)] for k in range(4)]
        states += [mine[0], other[0], mine[1], other[1], mine[2], other[2], mine[3], other[3], mine[4], mine[5]]
    rows = [nsr.get(id(q), 1) for q, _ in states]
    assert len(states) == 30 and [sorted(rows[10 * c:10 * c + 10])[-2:] for c in range(3)] == [[15, 16]] * 3, rows
    n_sub = 60
    single, alone = _engine(blob, 1), []
    try:
        for q, v in states:
            single.set_state(q[None], v[None])
            single.move_group("All", _targets(q[None]), 1e-9, n_sub)
            assert single.run() == 0
            gq, gv = single.get_state()
            alone.append((gq.cpu().numpy()[0].copy(), gv.cpu().numpy()[0].copy(), int(single.status()[0])))
    finally:
        single.close()
    q = np.stack([s[0] for s in states])
    v = np.stack([s[1] for s in states])
    eng = _engine(blob, 30, GE_MAXCTAS=1)
    try:
        assert eng.size(8) == 10
        eng.set_state(q, v)
        eng.move_group("All", _targets(q), 1e-9, n_sub)
        assert eng.run() == 0
        gq, gv = (x.cpu().numpy() for x in eng.get_state())
        st = eng.status().cpu().numpy()
    finally:
        eng.close()
    for e in range(30):
        aq, av, ast = alone[e]
        assert np.array_equal(gq[e], aq) and np.array_equal(gv[e], av) and int(st[e]) == ast, e
