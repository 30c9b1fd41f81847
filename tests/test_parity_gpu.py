"""GPU parity tests proper: the CUDA engine (through the C-ABI) against the fp64 CPU oracle on identical inputs.

Tolerances: both sides compute in fp64 with the same algorithms, so per-stage agreement is expected at rounding level
(1e-9 absolute is the gate); trajectories are compared at 1e-6 over hundreds of sub-steps (contact dynamics amplify
rounding differences) and the north-star tolerance (joint angles 1e-4, flags bit-exact) over whole grasp attempts.
"""
import numpy as np
import pytest

from tests.common import HOME, object_positions, reset_qpos_scene_a

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine4(scene_a):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, A, names = scene_a
    eng = BatchedEngine(blob, 4, 0)
    yield eng
    eng.close()


def _oracle(blob):
    from oracle.oracle_py import OracleEnv

    return OracleEnv(blob)


def _settled_states(scene_a, n, settle_steps):
    """n oracle envs reset by the scene-A rule and advanced settle_steps sub-steps; returns stacked (qpos, qvel, qacc_ws)."""
    blob, A, _ = scene_a
    out = []
    for i in range(n):
        o = _oracle(blob)
        o.reset(reset_qpos_scene_a(A, i))
        if settle_steps:
            o.move_group("All", None, 1e-7, settle_steps)
        out.append((o.qpos.copy(), o.qvel.copy()))
        o.close()
    return np.stack([s[0] for s in out]), np.stack([s[1] for s in out])


def test_library_reports_sm90(engine4):
    assert b"sm_90a" in engine4.L.ge_version()


@pytest.mark.parametrize("settle", [0, 150, 400])
def test_stage_parity(scene_a, engine4, settle):
    """kinematics, mass matrix, bias forces, contacts and the constraint solve of ONE forward pass, stage by stage"""
    blob, A, _ = scene_a
    qpos, qvel = _settled_states(scene_a, 4, settle)
    engine4.set_state(qpos, qvel)
    for env in range(4):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        o.forward()
        for field, ofield, tol in [("xpos", "xpos", 1e-12), ("xmat", "xmat", 1e-12), ("cdof", "cdof", 1e-12), ("qM", "qM", 1e-12),
                                   ("qfrc_bias", "qfrc_bias", 1e-10), ("qacc_smooth", "qacc_smooth", 1e-8)]:
            g = engine4.debug_forward(env, field)
            r = o.field(ofield)
            assert g.shape == r.shape, field
            scale = max(1.0, float(np.abs(r).max()))
            assert np.abs(g - r).max() <= tol * scale, (field, env, np.abs(g - r).max())
        ncon = int(engine4.debug_forward(env, "ncon")[0])
        assert ncon == o.ncon, (env, ncon, o.ncon)
        gc = engine4.debug_forward(env, "contact").reshape(-1, 16)
        oc = o.contacts()
        assert np.array_equal(gc[:, 13:], oc[:, 13:]), "contact geom ids / dims differ"
        assert np.abs(gc[:, :13] - oc[:, :13]).max(initial=0.0) < 1e-9
        for field in ("qacc", "qfrc_constraint"):
            g = engine4.debug_forward(env, field)
            r = o.field(field)
            scale = max(1.0, float(np.abs(r).max()))
            assert np.abs(g - r).max() <= 1e-7 * scale, (field, env, np.abs(g - r).max(), scale)
        o.close()


def test_substep_trajectory_parity(scene_a, engine4):
    """300 PID + mj_step sub-steps from the reset (objects dropping onto the table): qpos within 1e-6"""
    blob, A, _ = scene_a
    qpos, _ = _settled_states(scene_a, 4, 0)
    engine4.set_state(qpos)
    tgt = np.tile(HOME + np.array([0.3, 0.2, -0.2, 0.1, 0.1, 0.5, -0.1]), (4, 1))
    engine4.move_group("All", tgt, 1e-7, 300)
    assert engine4.run() == 0
    gq, gv = engine4.get_state()
    gq, gv = gq.cpu().numpy(), gv.cpu().numpy()
    res, steps, _, total = engine4.results()
    assert (res.cpu().numpy() == 2).all() and (steps.cpu().numpy() == 301).all()
    for env in range(4):
        o = _oracle(blob)
        o.reset(qpos[env])
        r, s = o.move_group("All", tgt[env], 1e-7, 300)
        assert (r, s) == (2, 301)
        assert np.abs(gq[env] - o.qpos).max() < 1e-6, (env, np.abs(gq[env] - o.qpos).max())
        assert np.abs(gv[env] - o.qvel).max() < 1e-4
        o.close()


def test_move_ee_parity(scene_a, engine4):
    """IK + Arm movement (MJ_Controller.move_ee): result code, step count identical, arm joints within 1e-6"""
    blob, A, _ = scene_a
    qpos, qvel = _settled_states(scene_a, 4, 500)
    engine4.set_state(qpos, qvel)
    targets = np.array([[0.0, -0.6, 1.1], [-0.15, -0.5, 1.1], [0.2, -0.7, 1.0], [0.6, 0.0, 1.15]])
    engine4.move_ee(targets, tolerance=0.05, max_steps=1000)
    assert engine4.run() == 0
    res, steps, _, _ = engine4.results()
    gq, _ = engine4.get_state()
    gq = gq.cpu().numpy()
    for env in range(4):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        r, s = o.move_ee(targets[env], 0.05, 1000)
        assert int(res[env]) == (r if r else 3) and int(steps[env]) == s, (env, int(res[env]), r, int(steps[env]), s)
        assert np.abs(gq[env][:8] - o.qpos[:8]).max() < 1e-6
        o.close()


def test_grasp_attempt_parity(scene_a, engine4):
    """whole move_and_grasp program on device vs oracle: reward bit-exact, per-phase step counts equal,
    arm joint angles within the north-star tolerance 1e-4"""
    blob, A, _ = scene_a
    qpos, qvel = _settled_states(scene_a, 4, 500)
    engine4.set_state(qpos, qvel)
    coords = np.zeros((4, 3))
    for env in range(4):
        p = object_positions(A, qpos[env])[env % 3]  # aim at one of the boxes
        coords[env] = [p[0], p[1], p[2] + 0.02]
    rot = np.array([0, 1, 3, 5], dtype=np.int32)
    engine4.grasp(coords, rot, 0.91)
    assert engine4.run() == 0
    _, _, reward, _ = engine4.results()
    info = engine4.grasp_info().cpu().numpy()
    gq, _ = engine4.get_state()
    gq = gq.cpu().numpy()
    for env in range(4):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        r, oinfo = o.move_and_grasp(coords[env], int(rot[env]), 0.91)
        assert int(reward[env]) == r, (env, int(reward[env]), r, info[env].tolist(), oinfo)
        assert info[env].tolist() == oinfo, (env, info[env].tolist(), oinfo)
        assert np.abs(gq[env][:8] - o.qpos[:8]).max() < 1e-4
        o.close()


def test_ik_and_pixel_2_world(scene_a, engine4):
    blob, A, _ = scene_a
    import torch

    xyz = np.array([[0, -0.6, 0.95], [0.1, -0.5, 1.0], [5, 5, 5], [-0.2, -0.7, 0.92]])
    q5, ok = engine4.ik(xyz)
    o = _oracle(blob)
    for i in range(4):
        r = o.ik(xyz[i])
        assert (r is not None) == bool(ok[i])
        if r is not None:
            assert np.abs(q5[i].cpu().numpy() - r).max() < 1e-12
    o.close()
    # media/console.png known answer (SURVEY 8c.1), default scene table height: depth 1.11 at pixel (136, 80)
    px = torch.tensor([136, 0, 199, 100], dtype=torch.int32)
    py = torch.tensor([80, 0, 199, 100], dtype=torch.int32)
    d = torch.tensor([1.11, 1.0, 1.0, 2.0], dtype=torch.float32)
    w = engine4.pixel_2_world(px, py, d).cpu().numpy()
    assert np.abs(w[0] - [-0.16551974, -0.50804459, 0.88999999]).max() < 1e-6


def test_render_parity(scene_a, engine4):
    """200x200 top-down RGB-D vs the oracle's ray caster: depth within 1e-4 m on >= 99.9 % of the pixels, rgb within 1 level"""
    blob, A, _ = scene_a
    qpos, qvel = _settled_states(scene_a, 4, 500)
    engine4.set_state(qpos, qvel)
    rgb, depth = engine4.render(1, 200, 200)
    rgb, depth = rgb.cpu().numpy(), depth.cpu().numpy()
    for env in range(2):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        orgb, odepth = o.render(1, 200, 200)
        close = np.abs(depth[env] - odepth) < 1e-4
        assert close.mean() >= 0.999, close.mean()
        assert (np.abs(rgb[env].astype(int) - orgb.astype(int)).max(axis=2)[close] <= 1).mean() > 0.999
        o.close()


def test_every_launch_gives_each_busy_env_its_whole_budget(scene_a):
    """ge_run_async(n) advances every busy environment by exactly n sub-steps, however its visits were spread over warps (with fewer
    envs than warp slots the next visit of an env is drawn while the previous one still runs), so the state after a sequence of
    launches does not depend on timing; and cutting the same iterations into launches differently gives bit-identical states"""
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, A, _ = scene_a
    n = 64
    q0 = np.stack([reset_qpos_scene_a(A, i) for i in range(n)])
    states = []
    for cuts in ((256,), (256,), (32,) * 8, (100, 156)):
        eng = BatchedEngine(blob, n, 0)
        eng.set_state(q0)
        eng.stay(20000)  # 10 000 sub-steps of holding still: busy through the whole test
        for c in cuts:
            eng.run_async(c)
        total = eng.results()[3].cpu().numpy()
        assert (eng.busy().cpu().numpy() != 0).all()
        assert (total == 256).all(), np.unique(total)
        qpos, qvel = eng.get_state()
        states.append((qpos.cpu().numpy(), qvel.cpu().numpy()))
        eng.close()
    for qpos, qvel in states[1:]:
        assert np.array_equal(qpos, states[0][0]) and np.array_equal(qvel, states[0][1])
