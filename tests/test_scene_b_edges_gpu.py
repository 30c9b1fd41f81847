"""The CTA-per-env build (scene B: the reference's default 40-object scene) at its capacity edges, against the fp64 oracle.

Fixture states: tests/golden/scene_b_edges.npz (tests/golden/make_scene_b_edges_golden.py: settling piles of eight resets and the
descent of a grasp attempt, chosen for many contacts, many and large contact islands).  Covered here:
  * the Hessian overflow row: with GE_HCAP at its minimum (Σ tree blocks + 6 maxcon + 64) every build with a large island moves its
    blocks to the env's row in HBM; the results must be the oracle's and bit-identical to the default region, for one env, for 8 envs
    in any order through k_run, and for a whole grasp attempt;
  * islands dealt to the 4 warps of the CTA: the layout of the last Newton Hessian build ("hlayout") is checked for consistency;
  * the contact list at its capacity (GE_MAXCON): the kept contacts are the oracle's first maxcon, status bit 0 is set iff more
    were found.
Stage tolerances as tests/test_scene_b_gpu.py: contacts 1e-7 (MPR stops at opt.mpr_tolerance), qacc / qfrc_constraint 1e-6 x scale.
"""
import os

import numpy as np
import pytest

from tests.common import HOME, contact_is_analytic, reset_qpos_scene_b

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scene_b_edges.npz")
NW = 4  # warps per CTA of the big-scene build
MAXCON = 112  # its default contact capacity


def _engine(blob, n, **env):
    """BatchedEngine with GE_* overrides set for ge_create only"""
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        return BatchedEngine(blob, n, 0)
    finally:
        for k in env:
            del os.environ[k]


def _need_min(A, maxcon=MAXCON):
    tdn = np.asarray(A["tree_dofnum"]).ravel().astype(int)
    nv = int(np.asarray(A["nv"]).ravel()[0])
    return min(int((tdn * (tdn + 1) // 2).sum()) + 6 * maxcon + 64, nv * (nv + 1) // 2)


def _hlayout(eng, env):
    h = eng.debug_forward(env, "hlayout")
    assert len(h) >= 3, "no Newton Hessian build"
    nt = int(h[2])
    t = h[3:3 + 5 * nt].reshape(nt, 5).astype(np.int64)
    return {"hflag": int(h[0]), "total": int(h[1]), "coupled": t[:, 0].astype(bool), "island": t[:, 1], "owner": t[:, 2],
            "offset": t[:, 3], "rows": t[:, 4]}


def _islands(lay):
    """{label: member trees} of the coupled trees"""
    out = {}
    for t in np.flatnonzero(lay["coupled"]):
        out.setdefault(int(lay["island"][t]), []).append(int(t))
    return out


def _debug(eng, env, fields=("qacc", "qfrc_constraint", "contact", "ncon", "ncand", "nmpr", "status", "hlayout")):
    return {f: eng.debug_forward(env, f) for f in fields}


@pytest.fixture(scope="module")
def fix():
    d = np.load(FIXTURE)
    return {k: d[k] for k in d.files}


@pytest.fixture(scope="module")
def oracle_ref(scene_b, fix):
    """oracle forward() of every fixture state: qacc, qfrc_constraint, contacts"""
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(scene_b[0])
    out = []
    for q, v in zip(fix["qpos"], fix["qvel"]):
        o.reset(q, v)
        o.forward()
        out.append({"qacc": o.field("qacc"), "qfrc_constraint": o.field("qfrc_constraint"), "contact": o.contacts(), "ncon": o.ncon})
    o.close()
    return out


def _check_oracle(g, r, what):
    gc, oc = g["contact"].reshape(-1, 16), r["contact"]
    assert gc.shape == oc.shape, (what, gc.shape, oc.shape)
    assert np.array_equal(gc[:, 13:], oc[:, 13:]), (what, "contact geom ids / dims differ")
    assert np.abs(gc[:, :13] - oc[:, :13]).max(initial=0.0) < 1e-7, what
    for f in ("qacc", "qfrc_constraint"):
        scale = max(1.0, float(np.abs(r[f]).max()))
        err = float(np.abs(g[f] - r[f]).max())
        assert err <= 1e-6 * scale, (what, f, err, scale)


def _check_layout(lay, hcap, hfull, tdn, what):
    """consistency of one Newton Hessian build's layout"""
    nt = len(tdn)
    isl = _islands(lay)
    for lab, members in isl.items():
        assert lab == min(members) and lay["island"][lab] == lab, (what, lab, members)
        owners = {int(lay["owner"][t]) for t in members}
        assert len(owners) == 1 and 0 <= owners.pop() < NW, (what, "owner", lab, lay["owner"][members])
        n = int(tdn[members].sum())
        assert all(lay["rows"][t] == n for t in members), (what, "island size", lab)
        assert all(lay["offset"][t] == lay["offset"][lab] for t in members), (what, "island offset", lab)
    for t in range(nt):
        if not lay["coupled"][t]:
            assert lay["island"][t] == t and lay["owner"][t] == -1 and lay["rows"][t] == tdn[t], (what, "uncoupled tree", t)
    # one block per uncoupled tree / per island (at its representative), back to back in ascending tree order
    off = 0
    for t in range(nt):
        if lay["coupled"][t] and lay["island"][t] != t:
            continue
        assert lay["offset"][t] == off, (what, "block offset", t, lay["offset"][t], off)
        n = int(lay["rows"][t])
        off += n * (n + 1) // 2
    assert off == lay["total"], (what, off, lay["total"])
    assert lay["hflag"] == int(lay["total"] > hcap), (what, lay["hflag"], lay["total"], hcap)
    assert lay["total"] <= (hfull if lay["hflag"] else hcap), what


def test_fixture_states_reach_the_capacity_edges(fix):
    """what the fixture was chosen for (the generator's contact graph, an upper bound of the engine's islands)"""
    assert len(fix["qpos"]) >= 10
    assert fix["ncomp"].max() > NW
    assert (fix["largest"] >= 42).sum() >= 3
    assert (fix["arm_in_largest"] == 1).any()
    assert fix["uncoupled_tree_max_contacts"].max() <= 15


def test_overflow_row_matches_default_region_and_oracle(scene_b, fix, oracle_ref):
    """GE_HCAP = Σ tree blocks + 6 maxcon + 64: builds whose blocks exceed it run in the env's HBM row; same numbers as the default
    region, bit for bit, and as the oracle"""
    blob, A, _ = scene_b
    need = _need_min(A)
    lo, hi = _engine(blob, 1, GE_HCAP=need), _engine(blob, 1)
    try:
        assert lo.size(10) == need and hi.size(10) > need and lo.size(11) == hi.size(11) == 248 * 249 // 2
        assert lo.size(6) == hi.size(6) == MAXCON
        tdn = np.asarray(A["tree_dofnum"]).ravel().astype(int)
        n_ovf, report = 0, []
        for s, (q, v) in enumerate(zip(fix["qpos"], fix["qvel"])):
            lo.set_state(q[None], v[None])
            hi.set_state(q[None], v[None])
            g_lo, g_hi = _debug(lo, 0), _debug(hi, 0)
            lay_lo, lay_hi = _hlayout(lo, 0), _hlayout(hi, 0)
            _check_layout(lay_lo, need, lo.size(11), tdn, ("min cap", s))
            _check_layout(lay_hi, hi.size(10), hi.size(11), tdn, ("default cap", s))
            n_ovf += lay_lo["hflag"]
            report.append((s, lay_lo["total"], lay_lo["hflag"], lay_hi["hflag"]))
            for f in g_lo:  # (hlayout: everything but hflag)
                assert np.array_equal(g_lo[f][f == "hlayout":], g_hi[f][f == "hlayout":]), (s, f)
            assert int(g_lo["status"][0]) == 0, (s, g_lo["status"])
            _check_oracle(g_lo, oracle_ref[s], s)
        print("state, block doubles, hflag at %d, hflag at %d:" % (need, hi.size(10)), report)
        assert n_ovf >= 3, report
    finally:
        lo.close()
        hi.close()


def _eight(fix):
    """the 8 fixture states with the largest block sums"""
    return np.argsort(-fix["blocks"], kind="stable")[:8]


def test_overflow_row_with_eight_envs_in_any_order(scene_b, fix):
    """8 envs, 8 different states, at the minimum region: every env's debug fields equal the state's in a 1-env engine, and 60 PID +
    mj_step sub-steps through k_run (8 CTAs at once, each with its own overflow row) equal the default region bit for bit, in two env
    orders"""
    blob, A, _ = scene_b
    need = _need_min(A)
    idx = _eight(fix)
    single = _engine(blob, 1, GE_HCAP=need)
    ref = {}
    try:
        for s in idx:
            single.set_state(fix["qpos"][s][None], fix["qvel"][s][None])
            ref[int(s)] = _debug(single, 0)
    finally:
        single.close()
    finals = []
    for order in (np.arange(8), np.array([5, 2, 7, 0, 3, 6, 1, 4])):
        states = idx[order]
        q, v = fix["qpos"][states], fix["qvel"][states]
        res = []
        for env in ({"GE_HCAP": need}, {}):
            eng = _engine(blob, 8, **env)
            try:
                eng.set_state(q, v)
                if env:
                    assert eng.size(10) == need
                    for e, s in enumerate(states):
                        g = _debug(eng, e)
                        for f in g:
                            assert np.array_equal(g[f], ref[int(s)][f]), (e, int(s), f)
                eng.move_group("All", None, 1e-7, 60)
                assert eng.run() == 0
                gq, gv = eng.get_state()
                res.append((gq.cpu().numpy().copy(), gv.cpu().numpy().copy(), eng.status().cpu().numpy().copy()))
            finally:
                eng.close()
        assert (res[0][2] == 0).all() and (res[1][2] == 0).all(), (res[0][2], res[1][2])
        assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
        finals.append({int(s): (res[0][0][e], res[0][1][e]) for e, s in enumerate(states)})
    for s in finals[0]:
        assert np.array_equal(finals[0][s][0], finals[1][s][0]) and np.array_equal(finals[0][s][1], finals[1][s][1]), s


def test_whole_grasp_attempt_through_the_overflow_row(scene_b):
    """tests/test_scene_b_gpu.py::test_scene_b_grasp_attempt_parity's attempt at the minimum region: reward, the 12 per-phase
    counters and the final state bit-identical to the default region"""
    from oracle.oracle_py import OracleEnv

    blob, A, _ = scene_b
    o = OracleEnv(blob)
    o.reset(reset_qpos_scene_b(A, 0))
    o.move_group("All", HOME + np.array([0, 0, 0, 0, 0, 0, 0.001]), 1e-9, 499)
    q, v = o.qpos.copy(), o.qvel.copy()
    o.close()
    pos = q[8:288].reshape(40, 7)[:, :3]
    on_table = (pos[:, 2] > 0.85) & (pos[:, 2] < 1.0)
    k = int((np.linalg.norm(pos[:, :2] - np.array([0.0, -0.6]), axis=1) + (~on_table) * 10).argmin())
    coords = np.array([pos[k, 0], pos[k, 1], pos[k, 2] + 0.02])
    out = []
    for env in ({"GE_HCAP": _need_min(A)}, {}):
        eng = _engine(blob, 1, **env)
        try:
            eng.set_state(q[None], v[None])
            eng.grasp(coords[None], np.array([1], dtype=np.int32), 0.91)
            assert eng.run() == 0
            _, _, reward, nsub = eng.results()
            gq, gv = eng.get_state()
            out.append((int(reward[0]), eng.grasp_info().cpu().numpy()[0].tolist(), int(nsub[0]), gq.cpu().numpy()[0].copy(),
                        gv.cpu().numpy()[0].copy(), int(eng.status()[0])))
        finally:
            eng.close()
    (r0, i0, n0, q0, v0, s0), (r1, i1, n1, q1, v1, s1) = out
    assert (r0, i0, n0, s0) == (r1, i1, n1, s1), ((r0, i0, n0, s0), (r1, i1, n1, s1))
    assert s0 == 0
    assert np.array_equal(q0, q1) and np.array_equal(v0, v1)


def test_islands_dealt_to_the_warps(scene_b, fix, oracle_ref):
    """default region: the states reach more islands than warps and an island of >= 30 dofs; every build's layout is consistent
    (owners in [0, 4) shared by an island, island size = its members' dofs, disjoint ascending blocks inside the region or the
    overflow row); qacc / qfrc_constraint as the oracle's"""
    blob, A, _ = scene_b
    tdn = np.asarray(A["tree_dofnum"]).ravel().astype(int)
    eng = _engine(blob, 1)
    try:
        hcap, hfull = eng.size(10), eng.size(11)
        most, largest, report = 0, 0, []
        for s, (q, v) in enumerate(zip(fix["qpos"], fix["qvel"])):
            eng.set_state(q[None], v[None])
            lay = _hlayout(eng, 0)
            _check_layout(lay, hcap, hfull, tdn, s)
            isl = _islands(lay)
            sizes = sorted((int(tdn[m].sum()) for m in isl.values()), reverse=True)
            # a coupled tree alone in its island took the coupled path for its number of contacts (> 15), not for a coupling
            lone = [m[0] for m in isl.values() if len(m) == 1]
            report.append((s, len(isl), sizes[:1], lay["total"], lay["hflag"], lone, sorted(set(lay["owner"][lay["coupled"]].tolist()))))
            most, largest = max(most, len(isl)), max(largest, sizes[0] if sizes else 0)
            _check_oracle(_debug(eng, 0, ("qacc", "qfrc_constraint", "contact")), oracle_ref[s], s)
        print("state, islands, largest island dofs, block doubles, hflag, lone coupled trees, owners:", report)
        assert most > NW and largest >= 30, (most, largest)
    finally:
        eng.close()


def _capacity_states(fix):
    """most contacts, the earliest state with contacts, the state of the descent with the most contacts, the state with the most
    analytic contacts beyond half its candidates"""
    desc = np.flatnonzero(fix["source"] > 0)
    room = fix["nanalytic"] - np.maximum(16, (fix["ncand"] + 1) // 2)
    return sorted({int(fix["ncon"].argmax()), int(np.argmin(np.where(fix["ncon"] > 0, fix["step"] + 10000 * fix["source"], 1 << 30))),
                   int(desc[fix["ncon"][desc].argmax()]), int(room.argmax())})


def _boxes_on_the_floor(A):
    """the ten box objects lying flat on the floor plane, apart (4 analytic contacts from one candidate pair each), every other object
    parked far apart in the air: 40 contacts from 10 candidates, so a capacity of 16 ends inside the analytic contacts without cutting
    the candidate list (no pile of the fixture has that many contacts per candidate)"""
    size = np.asarray(A["geom_size"]).reshape(-1, 3)
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(40):
        q[8 + 7 * i:15 + 7 * i] = [3.0 + i, 5.0, 6.0, 1, 0, 0, 0]
    for j in range(10):  # objects 10-19 are the boxes (geoms 40-49)
        q[8 + 7 * (10 + j):15 + 7 * (10 + j)] = [0.5 * j - 2.0, 3.0, size[40 + j, 2] - 0.0005, 1, 0, 0, 0]
    return q


def test_contact_list_at_capacity(scene_b, fix):
    """GE_MAXCON at ncon (exactly full), ncon - 1 and 16 (overflow) and inside the MPR section where earlier MPR pairs missed: the
    engine keeps the oracle's first maxcon contacts, sets status bit 0 iff more were found, never bit 64, and qacc is the capped
    oracle's.  Caps whose candidate list (2 maxcon) would be cut are checked only for bit 0 and a finite qacc.  Fixture states plus
    one built state (boxes on the floor) whose list overflows inside the analytic contacts."""
    from oracle.oracle_py import OracleEnv

    blob, A, _ = scene_b
    base = _engine(blob, 1)
    o = OracleEnv(blob)
    checked, truncated, inside, analytic, report = 0, 0, 0, 0, []
    try:
        for s in range(len(fix["qpos"])):  # nmpr at the default capacity, for every state
            base.set_state(fix["qpos"][s][None], fix["qvel"][s][None])
            report.append((s, int(base.debug_forward(0, "ncon")[0]), int(base.debug_forward(0, "ncand")[0]), int(base.debug_forward(0, "nmpr")[0])))
        print("state, ncon, ncand, nmpr at maxcon %d:" % MAXCON, report)
        cases = [(s, fix["qpos"][s], fix["qvel"][s]) for s in _capacity_states(fix)]
        cases.append(("boxes on the floor", _boxes_on_the_floor(A), np.zeros(248)))
        for s, q, v in cases:
            base.set_state(q[None], v[None])
            total, ncand, nmpr = (int(base.debug_forward(0, f)[0]) for f in ("ncon", "ncand", "nmpr"))
            assert total < MAXCON and int(base.debug_forward(0, "status")[0]) == 0
            o.set_maxcon(256)
            o.reset(q, v)
            o.forward()
            assert o.ncon == total
            n_an = int(contact_is_analytic(A, o.contacts()).sum())
            assert ncand == o.ncand, (s, ncand, o.ncand)
            caps = [total, total - 1, 16]
            if nmpr > total - n_an and total - n_an >= 2:  # some MPR pairs miss: a cap halfway through the MPR hits
                caps.append(n_an + (total - n_an) // 2)
                inside += 1
            cap_a = max(16, (ncand + 1) // 2)
            if cap_a < n_an:  # the list overflows inside the analytic contacts, the candidate list is not cut
                caps.append(cap_a)
                analytic += 1
            for cap in dict.fromkeys(caps):
                if cap < 16:
                    continue
                eng = _engine(blob, 1, GE_MAXCON=cap)
                try:
                    assert eng.size(6) == cap
                    eng.set_state(q[None], v[None])
                    g = _debug(eng, 0, ("contact", "ncon", "status", "qacc", "ncand"))
                finally:
                    eng.close()
                st = int(g["status"][0])
                assert not st & 64, (s, cap, st)
                assert np.isfinite(g["qacc"]).all(), (s, cap)
                assert int(g["ncand"][0]) == ncand
                if 2 * cap < ncand:  # the candidate list is cut too: which contacts exist legitimately differs from the oracle's
                    assert st & 1, (s, cap, st)
                    truncated += 1
                    continue
                o.set_maxcon(cap)
                o.reset(q, v)
                o.forward()
                assert o.con_overflow == int(total > cap)
                assert int(g["ncon"][0]) == min(total, cap) == o.ncon, (s, cap, int(g["ncon"][0]), total)
                assert (st & 1) == int(total > cap), (s, cap, st, total)
                gc, oc = g["contact"].reshape(-1, 16), o.contacts()
                assert np.array_equal(gc[:, 13:], oc[:, 13:]), (s, cap, "contacts are not the oracle's first maxcon")
                assert np.abs(gc[:, :13] - oc[:, :13]).max(initial=0.0) < 1e-7, (s, cap)
                r = o.field("qacc")
                assert np.abs(g["qacc"] - r).max() <= 1e-6 * max(1.0, float(np.abs(r).max())), (s, cap)
                checked += 1
        assert checked >= 6 and truncated >= 1 and inside >= 2 and analytic >= 1, (checked, truncated, inside, analytic)
    finally:
        base.close()
        o.close()
