"""The warp-per-env build (scene A: the 6-object scene) at its capacity edges, against the fp64 oracle.

Fixture states: tests/golden/scene_a_edges.npz (tests/golden/make_scene_a_edges_golden.py: a tower of the three boxes with balls against
it, grasp descents onto it, six objects packed in a corner of the drop bin, a box jammed into that corner).  The warp-per-env workspace
holds a Newton Hessian region of hcap doubles (410 by default, 336 at the smallest GE_HCAP, 990 = the full triangle); a build whose
blocks need more runs in the env's HBM overflow row, picked per warp (ten envs share one CTA).  Covered here:
  * three regions, one answer: contacts, qacc and qfrc_constraint equal the oracle's at every region and every debug field is
    bit-identical across the regions; the layout of the last Hessian build is consistent; ge_size(13) counts the overflowing builds;
  * the overflow decision at the region boundary (GE_HCAP = the build's block total, and one below);
  * ten envs in one CTA, several overflowing at once, through k_run: bit-identical to the same state alone and to the oracle's trajectory;
  * the contact list at its capacity (GE_MAXCON): the oracle's first maxcon contacts, status bit 0 iff more were found;
  * a whole grasp attempt whose fingers close on the middle box of the tower (arm + 3 objects: 414 doubles > 410).
Tolerances as tests/test_parity_gpu.py: analytic contacts 1e-9, MPR contacts 1e-7 (MPR stops at opt.mpr_tolerance), qacc /
qfrc_constraint 1e-6 x scale, counts, geom ids and dims exact.
"""
import os

import numpy as np
import pytest

from tests.common import contact_is_analytic, object_positions

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scene_a_edges.npz")
MAXCON = 32  # the warp-per-env build's default contact capacity on scene A
HCAP_MIN, HCAP_DEFAULT, HFULL = 336, 410, 990
FIELDS = ("qacc", "qfrc_constraint", "contact", "ncon", "niter", "nsr", "ncand", "nmpr", "status", "hlayout")


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


def _oracle(blob, maxcon=MAXCON):
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(blob)
    o.set_maxcon(maxcon)
    return o


def _hlayout(h):
    assert len(h) >= 3, "no Newton Hessian build"
    nt = int(h[2])
    t = h[3:3 + 5 * nt].reshape(nt, 5).astype(np.int64)
    return {"hflag": int(h[0]), "total": int(h[1]), "coupled": t[:, 0].astype(bool), "island": t[:, 1], "owner": t[:, 2],
            "offset": t[:, 3], "rows": t[:, 4]}


def _debug(eng, env=0, fields=FIELDS):
    return {f: eng.debug_forward(env, f) for f in fields}


def _same(a, b, what, skip_hflag=True):
    for f in a:
        x, y = a[f], b[f]
        if f == "hlayout" and skip_hflag:
            x, y = x[1:], y[1:]
        assert x.shape == y.shape and np.array_equal(x, y), (what, f)


@pytest.fixture(scope="module")
def fix():
    d = np.load(FIXTURE)
    return {k: d[k] for k in d.files}


def _check_oracle(A, g, o, what):
    """one engine forward() against the oracle's (contacts per kind, qacc / qfrc_constraint)"""
    oc = o.contacts()
    gc = g["contact"].reshape(-1, 16)
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
        assert err <= 1e-6 * scale, (what, f, err, scale)


def _check_layout(lay, hcap, tdn, what):
    """consistency of one Newton Hessian build's layout in the warp-per-env build (no owner warps: the env's warp does it all)"""
    nt = len(tdn)
    assert (lay["owner"] == -1).all(), (what, "owner", lay["owner"])
    isl = {}
    for t in np.flatnonzero(lay["coupled"]):
        isl.setdefault(int(lay["island"][t]), []).append(int(t))
    for lab, members in isl.items():
        assert lab == min(members) and lay["island"][lab] == lab, (what, lab, members)
        n = int(tdn[members].sum())
        assert all(lay["rows"][t] == n for t in members), (what, "island rows", lab)
        assert all(lay["offset"][t] == lay["offset"][lab] for t in members), (what, "island offset", lab)
    for t in range(nt):
        if not lay["coupled"][t]:
            assert lay["island"][t] == t and lay["rows"][t] == tdn[t], (what, "uncoupled tree", t)
    off = 0  # one block per uncoupled tree / per island (at its representative), back to back in ascending tree order
    for t in range(nt):
        if lay["coupled"][t] and lay["island"][t] != t:
            continue
        assert lay["offset"][t] == off, (what, "block offset", t, lay["offset"][t], off)
        n = int(lay["rows"][t])
        off += n * (n + 1) // 2
    assert off == lay["total"], (what, off, lay["total"])
    assert lay["hflag"] == int(lay["total"] > hcap), (what, lay["hflag"], lay["total"], hcap)
    return isl


def test_fixture_states_reach_the_capacity_edges(fix):
    """what the fixture was chosen for (the generator's contact graph, an upper bound of the engine's islands)"""
    b = fix["blocks"]
    assert len(b) >= 8
    assert ((b > HCAP_MIN) & (b <= HCAP_DEFAULT)).sum() >= 2  # (a) fit the default region, overflow the minimum one
    assert ((b > HCAP_DEFAULT) & (b <= 414)).sum() >= 2  # (b) arm + 3 objects, just above the default region
    assert b.max() == HFULL and fix["largest_trees"].max() == 7  # (c) one island of all seven trees
    mixed = (fix["nanalytic"] > 0) & (fix["nanalytic"] < fix["ncon"])
    assert fix["ncon"][mixed].max() >= 20 and (fix["ncon"] - fix["nanalytic"]).max() >= 4  # (d) analytic and MPR mixed
    assert fix["ncon"].max() > MAXCON  # a packed cluster beyond the default capacity
    assert fix["ncand"].max() <= 2 * MAXCON  # the default candidate list is never cut
    # (e) a box jammed into the drop bin's corner: the most contacts any scene-A state put on one uncoupled tree; the 8-lane group
    # path takes 15 (GE_TCAP), so a lone tree never takes the coupled path for its contact count
    assert fix["uncoupled_tree_max_contacts"].max() == 12


@pytest.mark.gpu
def test_three_regions_one_answer(scene_a, fix):
    """GE_HCAP = 336 (minimum), the default 410 and 990 (full triangle, no overflow row): contacts, qacc and qfrc_constraint equal
    the (32-contact) oracle's, every debug field is bit-identical across the regions, the hlayout is consistent, and ge_size(13)
    grows by 1..niter per forward() whose last build overflowed, never at 990"""
    blob, A, _ = scene_a
    tdn = np.asarray(A["tree_dofnum"]).ravel().astype(int)
    engs = [_engine(blob, 1, GE_HCAP=HCAP_MIN), _engine(blob, 1), _engine(blob, 1, GE_HCAP=HFULL)]
    o = _oracle(blob)
    try:
        assert [e.size(10) for e in engs] == [HCAP_MIN, HCAP_DEFAULT, HFULL]
        assert all(e.size(11) == HFULL and e.size(6) == MAXCON for e in engs)
        n_ovf, report = [0, 0, 0], []
        for s, (q, v) in enumerate(zip(fix["qpos"], fix["qvel"])):
            o.reset(q, v)
            o.forward()
            res = []
            for k, eng in enumerate(engs):
                eng.set_state(q[None], v[None])
                before = eng.size(13)
                h = eng.debug_forward(0, "hlayout")
                niter = int(eng.debug_forward(0, "niter")[0])  # (a second forward(): same build, same overflow)
                grew = eng.size(13) - before
                lay = _hlayout(h)
                isl = _check_layout(lay, eng.size(10), tdn, (s, k))
                # the two forward() calls each build the Hessian once per Newton iteration: their last build overflows iff hflag
                assert grew <= 2 * niter and (grew >= 2 or not lay["hflag"]) and (grew == 0 or k < 2), (s, k, lay["hflag"], grew, niter)
                n_ovf[k] += lay["hflag"]
                g = _debug(eng)
                st = int(g["status"][0])
                assert (st & 1) == int(fix["ncon"][s] > MAXCON) and not st & 64, (s, k, st)
                _check_oracle(A, g, o, (s, k))
                res.append(g)
            if fix["source"][s] == 4:  # the jammed box: 12 contacts on one tree that touches static geometry only
                assert not lay["coupled"].any() and int(res[1]["ncon"][0]) == fix["uncoupled_tree_max_contacts"][s]
            report.append((s, lay["total"], sorted(len(m) for m in isl.values()), [int(r["hlayout"][0]) for r in res]))
            _same(res[0], res[1], (s, "min / default"))
            _same(res[2], res[1], (s, "full / default"))
        print("state, block doubles, island sizes in trees, hflag at 336 / 410 / 990:", report)
        print("overflowing builds per region (336, 410, 990):", n_ovf)
        assert n_ovf[2] == 0 and n_ovf[1] >= 3 and n_ovf[0] > n_ovf[1], n_ovf
        assert engs[2].size(13) == 0
    finally:
        for e in engs:
            e.close()
        o.close()


@pytest.mark.gpu
def test_overflow_boundary(scene_a, fix):
    """the states of block sums 378 and 414: GE_HCAP = the build's block total keeps the blocks in shared memory (hflag 0), one
    below moves them to the overflow row (hflag 1); both bit-identical to the default region"""
    blob, A, _ = scene_a
    ref = _engine(blob, 1)
    checked = []
    try:
        for s in np.flatnonzero((fix["blocks"] > HCAP_MIN) & (fix["blocks"] <= 414)):
            q, v = fix["qpos"][s], fix["qvel"][s]
            ref.set_state(q[None], v[None])
            g_ref = _debug(ref)
            total = _hlayout(g_ref["hlayout"])["total"]
            for cap in (total, total - 1):
                if not HCAP_MIN <= cap <= HFULL:
                    continue
                eng = _engine(blob, 1, GE_HCAP=cap)
                try:
                    assert eng.size(10) == cap
                    eng.set_state(q[None], v[None])
                    g = _debug(eng)
                finally:
                    eng.close()
                assert int(g["hlayout"][0]) == int(cap < total), (int(s), cap, total, int(g["hlayout"][0]))
                _same(g, g_ref, (int(s), cap))
                checked.append((int(s), cap, int(g["hlayout"][0])))
    finally:
        ref.close()
    print("state, GE_HCAP, hflag:", checked)
    assert sum(c[2] for c in checked) >= 3 and sum(1 - c[2] for c in checked) >= 3, checked


def _thirty(fix):
    """30 envs: every fixture state three times, interleaved"""
    n = len(fix["qpos"])
    return np.array([i % n for i in range(30)])


def _targets(q):
    """a small movement of every joint from where it stands: the PID keeps pushing through all 60 sub-steps"""
    return q[:, :7] + np.array([0.02, -0.02, 0.02, 0.01, 0.01, 0.05, 0.0])


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [{"GE_MAXCTAS": 1}, {"GE_MAXCTAS": 2, "GE_WPB": 5}], ids=["1x10", "2x5"])
def test_ten_envs_in_one_cta(scene_a, fix, shape):
    """30 envs, every fixture state three times, through k_run with one CTA of ten warps (or two of five): each warp takes several
    envs and several overflow at once.  60 PID + sub-steps at the minimum and the default region, in two env orders: each env's final
    qpos, qvel and status are bit-identical to the state alone in a 1-env engine, and within 1e-6 of the oracle"""
    blob, A, _ = scene_a
    n_sub = 60
    states = np.arange(len(fix["qpos"]))
    single, alone = _engine(blob, 1), {}
    try:
        for s in states:
            q, v = fix["qpos"][s][None], fix["qvel"][s][None]
            single.set_state(q, v)
            single.move_group("All", _targets(q), 1e-9, n_sub)
            assert single.run() == 0
            gq, gv = single.get_state()
            alone[int(s)] = (gq.cpu().numpy()[0].copy(), gv.cpu().numpy()[0].copy(), int(single.status()[0]))
    finally:
        single.close()
    o = _oracle(blob)
    for s in states:  # the oracle's trajectory, 32 contacts per sub-step as the engine
        o.reset(fix["qpos"][s], fix["qvel"][s])
        r, _ = o.move_group("All", _targets(fix["qpos"][s][None])[0], 1e-9, n_sub)
        assert r == 2
        gq, gv, st = alone[int(s)]
        assert np.abs(gq - o.qpos).max() < 1e-6, (int(s), np.abs(gq - o.qpos).max())
        assert np.abs(gv - o.qvel).max() < 1e-4, (int(s), np.abs(gv - o.qvel).max())
        assert (st & 1) == int(fix["ncon"][s] > MAXCON) and not (st & ~5), (int(s), st)
    o.close()
    idx = _thirty(fix)
    rng = np.random.RandomState(7)
    for order in (np.arange(30), rng.permutation(30)):
        sel = idx[order]
        q, v = fix["qpos"][sel], fix["qvel"][sel]
        for region in ({"GE_HCAP": HCAP_MIN}, {}):
            eng = _engine(blob, 30, **shape, **region)
            try:
                assert eng.size(8) == (10 if shape["GE_MAXCTAS"] == 1 else 5)
                eng.set_state(q, v)
                eng.move_group("All", _targets(q), 1e-9, n_sub)
                assert eng.run() == 0
                gq, gv = eng.get_state()
                gq, gv, st = gq.cpu().numpy(), gv.cpu().numpy(), eng.status().cpu().numpy()
                assert eng.size(13) > 0  # overflowing builds ran among the others
            finally:
                eng.close()
            for e, s in enumerate(sel):
                aq, av, ast = alone[int(s)]
                assert np.array_equal(gq[e], aq) and np.array_equal(gv[e], av) and int(st[e]) == ast, (shape, region, e, int(s))


def _capacity_states(fix):
    """the most contacts with analytic and MPR mixed, the most MPR contacts, and the packed bin corner (more than 32 contacts)"""
    mixed = np.flatnonzero((fix["nanalytic"] > 0) & (fix["nanalytic"] < fix["ncon"]))
    return sorted({int(mixed[fix["ncon"][mixed].argmax()]), int((fix["ncon"] - fix["nanalytic"]).argmax()), int(fix["ncon"].argmax())})


@pytest.mark.gpu
def test_contact_list_at_capacity(scene_a, fix):
    """GE_MAXCON at ncon (exactly full), ncon - 1 and 16, inside the MPR contacts where earlier MPR pairs missed, and inside the
    analytic contacts: the engine keeps the oracle's first maxcon contacts, sets status bit 0 iff more were found, never bit 64, and
    qacc is the capped oracle's.  Caps whose candidate list (2 maxcon) would be cut are checked only for bit 0 and a finite qacc.  The
    state beyond 32 contacts is also checked at the default capacity."""
    from oracle.oracle_py import OracleEnv

    blob, A, _ = scene_a
    base = _engine(blob, 1, GE_MAXCON=64)
    o = OracleEnv(blob)
    checked, truncated, inside, analytic, default_cap, report = 0, 0, 0, 0, 0, []
    try:
        assert base.size(6) == 64
        for s in _capacity_states(fix):
            q, v = fix["qpos"][s], fix["qvel"][s]
            base.set_state(q[None], v[None])
            total, ncand, nmpr = (int(base.debug_forward(0, f)[0]) for f in ("ncon", "ncand", "nmpr"))
            assert total < 64 and int(base.debug_forward(0, "status")[0]) == 0
            o.set_maxcon(256)
            o.reset(q, v)
            o.forward()
            assert o.ncon == total and ncand == o.ncand, (s, total, o.ncon, ncand, o.ncand)
            n_an = int(contact_is_analytic(A, o.contacts()).sum())
            report.append((s, total, n_an, ncand, nmpr))
            caps = [total, total - 1, 16]
            if nmpr > total - n_an and total - n_an >= 2:  # some MPR pairs miss: a cap halfway through the MPR hits
                caps.append(n_an + (total - n_an) // 2)
                inside += 1
            cap_a = max(16, (ncand + 1) // 2)
            if cap_a < n_an:  # the list overflows inside the analytic contacts, the candidate list is not cut
                caps.append(cap_a)
                analytic += 1
            if total > MAXCON:
                caps.append(None)  # the default capacity, without GE_MAXCON
                default_cap += 1
            for cap in dict.fromkeys(caps):
                if cap is not None and cap < 16:
                    continue
                eng = _engine(blob, 1, **({} if cap is None else {"GE_MAXCON": cap}))
                cap = cap or MAXCON
                try:
                    assert eng.size(6) == cap
                    eng.set_state(q[None], v[None])
                    g = _debug(eng, 0, ("contact", "ncon", "status", "qacc", "qfrc_constraint", "ncand"))
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
                _check_oracle(A, g, o, (s, cap))
                checked += 1
        print("state, ncon, analytic, ncand, nmpr at maxcon 64:", report)
        assert checked >= 8 and inside >= 1 and analytic >= 1 and default_cap >= 1, (checked, truncated, inside, analytic, default_cap)
    finally:
        base.close()
        o.close()


@pytest.mark.gpu
def test_whole_grasp_attempt_through_a_large_island(scene_a, fix):
    """a scripted attempt whose fingers close on box_1, in the middle of the tower (it touches box_3 below and box_2 above): arm +
    3 objects = 414 doubles, over the default region.  Reward and the 12 phase counters equal the oracle's, arm angles within 1e-4, and
    everything bit-identical at the minimum, default and full region"""
    blob, A, _ = scene_a
    s = int(np.flatnonzero((fix["source"] == 0) & (fix["step"] == 0) & (fix["blocks"] < 400) & (fix["largest_trees"] == 4))[0])
    q, v = fix["qpos"][s], fix["qvel"][s]  # the placed tower with one ball against its foot
    p = object_positions(A, q)[0]
    coords = np.array([p[0], p[1], p[2] + 0.02])
    o = _oracle(blob)
    o.reset(q, v)
    r, oinfo = o.move_and_grasp(coords, 1, 0.91)
    oq = o.qpos.copy()
    o.close()
    out = []
    for region in ({"GE_HCAP": HCAP_MIN}, {}, {"GE_HCAP": HFULL}):
        eng = _engine(blob, 1, **region)
        try:
            eng.set_state(q[None], v[None])
            eng.grasp(coords[None], np.array([1], dtype=np.int32), 0.91)
            assert eng.run() == 0
            _, _, reward, nsub = eng.results()
            gq, gv = eng.get_state()
            out.append((int(reward[0]), eng.grasp_info().cpu().numpy()[0].tolist(), int(nsub[0]), int(eng.status()[0]),
                        gq.cpu().numpy()[0].copy(), gv.cpu().numpy()[0].copy(), eng.size(13)))
        finally:
            eng.close()
    print("reward, phase counters, sub-steps, status, overflowing builds at 336 / 410 / 990:", [x[:4] + x[6:] for x in out])
    for reward, info, nsub, st, gq, gv, _ in out:
        assert (reward, info) == (r, oinfo), (reward, info, r, oinfo)
        assert st == 0
        assert np.abs(gq[:8] - oq[:8]).max() < 1e-4
    for x in out[1:]:
        assert x[:4] == out[0][:4] and np.array_equal(x[4], out[0][4]) and np.array_equal(x[5], out[0][5])
    assert out[1][6] > 0 and out[2][6] == 0 and out[0][6] >= out[1][6]  # the fingers' island did overflow the default region
