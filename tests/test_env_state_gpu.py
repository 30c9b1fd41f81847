"""Environment state records on the device (ge_snapshot / ge_restore / ge_clone, BatchedEngine and BatchedGraspEnv on top of them):
bit-exact save and resume, mid-attempt included, copies between slots and engines, refusal of foreign or malformed records, the hand-off
to and from the fp64 oracle, and grasp labelling from branched copies of an env (evaluate_actions).

Engine tests run on scene A (warp-per-env build, workspace in shared memory) and scene B (CTA-per-env build) from the settled states of
tests/golden/success_64 and tests/golden/scene_b_attempts, with the grasps recorded there (scene B: only those, see DESIGN.md section 4).
"Bit-identical" compares the bytes of qpos, qvel, targets, controls, results, total sub-steps, grasp info, status, busy and the warm start
as the solver sees it (debug_forward(e, "qacc")), as tests/test_engine_commands_gpu.py does; the records themselves are compared too.
Hand-off gates are tests/test_parity_gpu.py's: reward and grasp info exact, the arm within 1e-4 over a whole attempt.
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = ("qpos", "qvel", "target", "ctrl", "result", "steps", "reward", "total", "info", "status", "busy", "qacc")
N = 8


def _engine(blob, n):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    return BatchedEngine(blob, n, 0)


def _fixture(scene):
    name = "success_64" if scene == "A" else "scene_b_attempts"
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    recs = json.load(open(os.path.join(GOLDEN, name + ".json")))["records"][:N]
    rot = [r["action"][1] if "action" in r else r["rot"] for r in recs]
    return z["qpos0"][:N], z["qvel0"][:N], np.array([r["coords"] for r in recs]), np.array(rot, np.int32)


@pytest.fixture(scope="module", params=["A", "B"])
def case(request, scene_a, scene_b):
    blob = (scene_a if request.param == "A" else scene_b)[0]
    return (request.param, blob) + _fixture(request.param)


def _snap(eng):
    qpos, qvel = eng.get_state()
    result, steps, reward, total = eng.results()
    s = {"qpos": qpos, "qvel": qvel, "target": eng.get_targets(), "ctrl": eng.get_ctrl(), "result": result, "steps": steps,
         "reward": reward, "total": total, "info": eng.grasp_info(), "status": eng.status(), "busy": eng.busy()}
    s = {k: v.cpu().numpy() for k, v in s.items()}
    s["qacc"] = np.stack([eng.debug_forward(e, "qacc") for e in range(eng.n_envs)])
    s["record"] = eng.snapshot().data.cpu().numpy()
    return s


def _same(a, b, ea, eb, what, keys=KEYS + ("record",)):
    for k in keys:
        assert a[k][ea].tobytes() == b[k][eb].tobytes(), (what, ea, eb, k, a[k][ea], b[k][eb])


def _all_same(a, b, what):
    for e in range(len(a["qpos"])):
        _same(a, b, e, e, what)


def _mid_attempt(eng, coords, rot, chunk=150):
    """grasp, then partial runs until the busy envs stand in at least two different program phases"""
    eng.grasp(coords, rot, 0.91)
    for _ in range(40):
        assert eng.run(max_substeps=chunk) > 0, "every attempt ended before the envs were spread over program phases"
        ph = eng.snapshot().field("prog_phase").cpu().numpy()
        if len(set(ph[ph != 0].tolist())) >= 2:
            return ph
    raise AssertionError("no two program phases at once")


def test_identity_and_record_size(case):
    from mujoco_rl_ur5_b200.env_state import record_size

    scene, blob, q0, v0, coords, rot = case
    eng = _engine(blob, N)
    assert eng.state_bytes == record_size(eng.nq, eng.nv) == {"A": 1536, "B": 6784}[scene]
    eng.set_state(q0, v0)
    eng.move_group("Arm", None, 1e-7, 30)
    eng.run()
    s = eng.snapshot()
    before = _snap(eng)
    eng.grasp(coords, rot, 0.91)
    assert eng.run() == 0
    assert _snap(eng)["total"].tolist() != before["total"].tolist()
    eng.restore(s)
    _all_same(before, _snap(eng), "restore all")
    eng.close()


def test_determinism_after_restore(case):
    scene, blob, q0, v0, coords, rot = case
    eng = _engine(blob, N)
    eng.set_state(q0, v0)
    s = eng.snapshot()
    runs = []
    for _ in range(2):
        eng.restore(s)
        eng.grasp(coords, rot, 0.91)
        assert eng.run() == 0
        runs.append(_snap(eng))
    _all_same(runs[0], runs[1], "attempt replayed after restore")
    assert (runs[0]["status"] == 0).all()
    eng.close()


def test_mid_attempt_resume_here_and_in_another_engine(case):
    scene, blob, q0, v0, coords, rot = case
    eng = _engine(blob, N)
    eng.set_state(q0, v0)
    ph = _mid_attempt(eng, coords, rot)
    s = eng.snapshot()
    mid = _snap(eng)
    assert mid["busy"].any()
    assert eng.run() == 0
    first = _snap(eng)
    eng.restore(s)
    _all_same(mid, _snap(eng), "mid-attempt restore")
    assert eng.run() == 0
    _all_same(first, _snap(eng), "finished again")
    eng.close()
    # the same records, scattered over a fresh engine of another size
    M = N + 5
    dest = np.random.default_rng(3).permutation(M)[:N]
    rows = np.full(M, -1, np.int32)
    rows[dest] = np.arange(N)
    other = _engine(blob, M)
    untouched = _snap(other)
    other.restore(s, rows)
    got = _snap(other)
    for e in range(N):
        _same(mid, got, e, dest[e], "scattered restore")
    for e in set(range(M)) - set(dest.tolist()):
        _same(untouched, got, e, e, "row -1")
    assert other.run() == 0
    got = _snap(other)
    for e in range(N):
        _same(first, got, e, dest[e], "finished in another engine")
    other.close()
    print(f"scene {scene}: phases at the snapshot {sorted(set(ph.tolist()))}")


def test_clone_maps(case):
    scene, blob, q0, v0, coords, rot = case
    eng = _engine(blob, N)
    eng.set_state(q0, v0)
    _mid_attempt(eng, coords, rot)
    s = eng.snapshot()
    for src in (np.arange(N)[::-1], np.full(N, 2), np.array([-1, 0, 0, 7, -1, 3, 6, -1])):
        eng.restore(s)
        before = _snap(eng)
        eng.clone(src.astype(np.int32))
        after = _snap(eng)
        for e in range(N):
            _same(before, after, src[e] if src[e] >= 0 else e, e, ("clone", src.tolist()))
    # identical grasps on clones of one idle source give identical records
    eng.set_state(q0, v0)
    eng.clone(np.full(N, 1, np.int32))
    eng.grasp(np.tile(coords[1], (N, 1)), np.full(N, rot[1], np.int32), 0.91)
    assert eng.run() == 0
    rec = eng.snapshot().data.cpu().numpy()
    assert all(rec[e].tobytes() == rec[0].tobytes() for e in range(N))
    eng.close()


def test_refusals_leave_the_engine_unchanged(case, scene_a, scene_b):
    from mujoco_rl_ur5_b200.engine import EngineError

    scene, blob, q0, v0, coords, rot = case
    eng = _engine(blob, N)
    eng.set_state(q0, v0)
    _mid_attempt(eng, coords, rot)
    before = _snap(eng)
    foreign = _engine((scene_b if scene == "A" else scene_a)[0], N)
    with pytest.raises(EngineError, match="bytes"):  # the other scene's records have another size
        eng.restore(foreign.snapshot())
    s = eng.snapshot()
    from mujoco_rl_ur5_b200.env_state import EngineState

    f = foreign.snapshot()
    same_size = EngineState(s.data.clone(), s.nq, s.nv, s.fingerprint)
    same_size.data[:, 8:16] = f.data[:, 8:16]  # another model's fingerprint in a record of the right size
    with pytest.raises(EngineError, match="\\(-4\\)"):
        eng.restore(same_size)
    bad = EngineState(s.data.clone(), s.nq, s.nv, s.fingerprint)
    bad.data[5, 0] ^= 1
    with pytest.raises(EngineError, match="\\(-4\\)"):
        eng.restore(bad)
    for r in (N, -2):
        rows = np.arange(N, dtype=np.int32)
        rows[3] = r
        with pytest.raises(EngineError, match="\\(-1\\)"):
            eng.restore(s, rows)
        with pytest.raises(EngineError, match="\\(-1\\)"):
            eng.clone(rows)
    with pytest.raises(EngineError, match="\\(-4\\)"):  # a record of an out-of-range snapshot index is all zeros
        eng.restore(eng.snapshot(np.array([0, N] + list(range(2, N)), np.int32)))
    _all_same(before, _snap(eng), "refused calls")
    foreign.close()
    eng.close()


def test_record_moves_between_the_warp_and_cta_builds(scene_a, monkeypatch):
    blob = scene_a[0]
    q0, v0, coords, rot = _fixture("A")
    eng = _engine(blob, N)
    eng.set_state(q0, v0)
    _mid_attempt(eng, coords, rot)
    s = eng.snapshot()
    monkeypatch.setenv("GE_CTA_PER_ENV", "1")
    hbm = _engine(blob, N)
    monkeypatch.delenv("GE_CTA_PER_ENV")
    assert eng.size(9) == 0 and hbm.size(9) == 1
    hbm.restore(s)
    assert hbm.snapshot().data.cpu().numpy().tobytes() == s.data.cpu().numpy().tobytes()
    hbm.close()
    eng.close()


def _handoff_gates(eng, o, coords, rot, e, sub0_gpu, what):
    from mujoco_rl_ur5_b200.engine import EngineError  # noqa: F401

    osub0 = o.substeps
    r, oinfo = o.move_and_grasp(coords[e], int(rot[e]), 0.91)
    _, _, reward, total = eng.results()
    info = eng.grasp_info().cpu().numpy()
    gq = eng.get_state()[0].cpu().numpy()
    assert int(reward[e]) == r and info[e].tolist() == oinfo, (what, e, int(reward[e]), r, info[e].tolist(), oinfo)
    assert int(total[e]) - sub0_gpu[e] == o.substeps - osub0, (what, e)
    assert np.abs(gq[e][:8] - o.qpos[:8]).max() < 1e-4, (what, e, np.abs(gq[e][:8] - o.qpos[:8]).max())


def test_oracle_handoff_both_directions(scene_a):
    from mujoco_rl_ur5_b200.env_state import CTL_CTRL, CTL_KP, CTL_LAST, CTL_TARGET, EngineState
    from oracle.oracle_py import OracleEnv
    from tests.common import HOME

    blob = scene_a[0]
    q0, v0, coords, rot = _fixture("A")
    n = 4
    q0, v0, coords, rot = q0[:n], v0[:n], coords[:n], rot[:n]
    tgt = np.tile(HOME + np.array([0.05, 0.1, -0.1, 0.05, 0.0, 0.3, 0.0]), (n, 1))
    # GPU -> oracle: after a movement with a changed gain, the warm start and the whole PID block are non-trivial
    eng = _engine(blob, n)
    eng.set_state(q0, v0)
    eng.set_gain(0, 12.5)
    eng.move_group("All", tgt, 1e-7, 120)
    eng.run()
    s = eng.snapshot()
    sub0 = eng.results()[3].cpu().numpy()
    eng.grasp(coords, rot, 0.91)
    assert eng.run() == 0
    for e in range(n):
        f = s.fields(e)
        assert np.abs(f["qaccws"]).max() > 0 and f["ctl"][CTL_KP] == 12.5
        o = OracleEnv(blob)
        o.reset(f["qpos"])
        o.qpos[:], o.qvel[:], o.qacc_warmstart[:] = f["qpos"], f["qvel"], f["qaccws"]
        ctl = f["ctl"]
        o.target[:], o.last_input[:], o.kp[:], o.ctrl[:] = ctl[CTL_TARGET:CTL_TARGET + 7], ctl[CTL_LAST:CTL_LAST + 7], ctl[CTL_KP:CTL_KP + 7], ctl[CTL_CTRL:CTL_CTRL + 7]
        o.fk()
        _handoff_gates(eng, o, coords, rot, e, sub0, "GPU -> oracle")
        o.close()
    # oracle -> GPU
    oracles, dicts = [], []
    for e in range(n):
        o = OracleEnv(blob)
        o.reset(q0[e], v0[e])
        o.kp[0] = 12.5
        o.move_group("All", tgt[e], 1e-7, 120)
        ctl = np.zeros(32)
        ctl[CTL_TARGET:CTL_TARGET + 7], ctl[CTL_LAST:CTL_LAST + 7], ctl[CTL_KP:CTL_KP + 7], ctl[CTL_CTRL:CTL_CTRL + 7] = o.target, o.last_input, o.kp, o.ctrl
        dicts.append({"qpos": o.qpos.copy(), "qvel": o.qvel.copy(), "qaccws": o.qacc_warmstart.copy(), "ctl": ctl, "substeps": o.substeps})
        oracles.append(o)
    rec = EngineState.from_fields(dicts, eng.fingerprint, eng.nq, eng.nv)
    eng.restore(rec)
    sub0 = eng.results()[3].cpu().numpy()
    assert sub0.tolist() == [d["substeps"] for d in dicts]
    eng.grasp(coords, rot, 0.91)
    assert eng.run() == 0
    for e, o in enumerate(oracles):
        _handoff_gates(eng, o, coords, rot, e, sub0, "oracle -> GPU")
        o.close()
    eng.close()


def _table_actions(env, rng, n, k):
    """pixels in the middle of the top-down image (mostly table and objects) and random rotations, [n, k, 2]"""
    W = env.IMAGE_WIDTH
    x, y = rng.integers(60, 140, (n, k)), rng.integers(60, 140, (n, k))
    return np.stack([y * W + x, rng.integers(0, 6, (n, k))], axis=-1).astype(np.int32)


def _env_bytes(env):
    return env.engine.snapshot().data.cpu().numpy().tobytes(), {k: v.cpu().numpy().tobytes() for k, v in env.current_observation.items()}


def test_evaluate_actions_matches_step():
    import torch

    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    # the settled success_64 states and their recorded grasps (mostly successful) in column 0, random table pixels in columns 1 and 2
    env = BatchedGraspEnv(N, "A")
    q0, v0, _, _ = _fixture("A")
    env.engine.set_state(q0, v0)
    env.current_observation = env.get_observation()
    s0 = env.snapshot()
    st0 = _env_bytes(env)
    golden = json.load(open(os.path.join(GOLDEN, "success_64.json")))["records"][:N]
    a3 = _table_actions(env, np.random.default_rng(7), N, 3)
    a3[:, 0] = [r["action"] for r in golden]
    # K = 1: the step's own reward, executed flag and grasp info
    r1, x1 = env.evaluate_actions(a3[:, :1])
    assert _env_bytes(env) == st0
    binfo = env._branch.grasp_info().cpu().numpy()
    _, rew, _, info = env.step(a3[:, 0])
    assert r1[:, 0].cpu().numpy().tolist() == rew.tolist() and torch.equal(x1[:, 0], info["executed"])
    assert binfo.tobytes() == env.engine.grasp_info().cpu().numpy().tobytes()
    assert x1.any(), "no attempt was executed"
    # K = 3: every column is a restore-then-step run of its action; chunked evaluation gives the same
    env.restore(s0)
    assert _env_bytes(env) == st0
    r3, x3 = env.evaluate_actions(a3)
    assert _env_bytes(env) == st0
    r3c, x3c = env.evaluate_actions(a3, max_branch_envs=5)
    assert torch.equal(r3, r3c) and torch.equal(x3, x3c)
    for k in range(3):
        env.restore(s0)
        _, rew, _, info = env.step(a3[:, k])
        assert r3[:, k].cpu().numpy().tolist() == rew.tolist() and torch.equal(x3[:, k], info["executed"]), k
    assert r3[:, 0].any(), "no recorded grasp succeeded"
    print(f"evaluate_actions: rewards {r3.cpu().numpy().tolist()}")
    env.close()


def test_facade_checkpoint_resumes_the_next_step(tmp_path):
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv
    from mujoco_rl_ur5_b200.engine import EngineError
    from mujoco_rl_ur5_b200.env_state import EngineState

    rng = np.random.default_rng(11)
    env = BatchedGraspEnv(N, "A")
    env.reset()
    env.step(_table_actions(env, rng, N, 1)[:, 0])
    p = str(tmp_path / "envs.pt")
    env.snapshot().save(p)
    a = _table_actions(env, rng, N, 1)[:, 0]
    other = BatchedGraspEnv(N, "A", seed_base=777)
    other.restore(EngineState.load(p))
    assert (other.step_called, other.episode) == (env.step_called, env.episode)
    o1, r1, _, _ = env.step(a)
    o2, r2, _, _ = other.step(a)
    assert r1.tolist() == r2.tolist()
    for k in ("rgb", "depth"):
        assert o1[k].cpu().numpy().tobytes() == o2[k].cpu().numpy().tobytes(), k
    assert _env_bytes(env) == _env_bytes(other)
    env.close()
    other.close()
    b = BatchedGraspEnv(N, "B")
    with pytest.raises(EngineError):
        b.restore(EngineState.load(p))
    assert b.step_called == 0 and b.current_observation is None
    b.close()
