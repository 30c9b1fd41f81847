"""Scene B (UR5gripper_2_finger_many_objects.xml: 40 free objects, condim-6 contacts, nv = 248 — the reference's DEFAULT scene,
GraspingEnv.py:30) on the CUDA engine against the fp64 oracle, plus the HBM-resident workspace path exercised with scene A.

Scene B does not fit the per-warp shared-memory workspace (the packed Newton Hessian alone is 247 KB), so the engine keeps one
workspace row per env in HBM (ge_size(9) == 1).  Tolerances as in test_parity_gpu.py: stage level 1e-9, short trajectories 1e-6.
"""
import os

import numpy as np
import pytest

from tests.common import HOME, reset_qpos_scene_a, reset_qpos_scene_b

pytestmark = pytest.mark.gpu


def _oracle(blob):
    from oracle.oracle_py import OracleEnv

    return OracleEnv(blob)


@pytest.fixture(scope="module")
def settled_b(scene_b):
    """two oracle envs: reset by the reference rule, then 0 / 400 sub-steps (free fall, impacts, pile forming) while the arm
    tracks an unreachable-within-tolerance target so that the movement never ends early"""
    blob, A, _ = scene_b
    out = {}
    for settle in (0, 400):
        qs, vs = [], []
        for i in range(2):
            o = _oracle(blob)
            o.reset(reset_qpos_scene_b(A, i))
            if settle:
                o.move_group("All", HOME + np.array([0.2, 0.1, -0.1, 0.1, 0.1, 0.3, -0.1]), 1e-7, settle)
            qs.append(o.qpos.copy()); vs.append(o.qvel.copy())
            o.close()
        out[settle] = (np.stack(qs), np.stack(vs))
    return out


@pytest.fixture(scope="module")
def engine_b(scene_b):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    eng = BatchedEngine(scene_b[0], 2, 0)
    yield eng
    eng.close()


def test_scene_b_uses_the_big_scene_build(engine_b):
    """ge_size(9) == 1: the CTA-per-env build (r01: HBM-row workspace; r02: one env per CTA of 4 warps, workspace in shared memory)"""
    assert engine_b.size(9) == 1 and engine_b.size(1) == 248 and engine_b.size(6) >= 96
    assert engine_b.size(7) <= 116736 - 1024  # two CTAs (= two envs) per SM


@pytest.mark.parametrize("settle", [0, 400])
def test_scene_b_stage_parity(scene_b, engine_b, settled_b, settle):
    blob, A, _ = scene_b
    qpos, qvel = settled_b[settle]
    engine_b.set_state(qpos, qvel)
    for env in range(2):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        o.forward()
        for field, tol in [("xpos", 1e-12), ("xmat", 1e-12), ("cdof", 1e-12), ("qM", 1e-12), ("qfrc_bias", 1e-10), ("qacc_smooth", 1e-8)]:
            g, r = engine_b.debug_forward(env, field), o.field(field)
            assert g.shape == r.shape, field
            assert np.abs(g - r).max() <= tol * max(1.0, float(np.abs(r).max())), (field, env, np.abs(g - r).max())
        assert int(engine_b.debug_forward(env, "ncon")[0]) == o.ncon, (env, o.ncon)
        if settle:
            assert o.ncon >= 20  # objects piling up on the table
        gc = engine_b.debug_forward(env, "contact").reshape(-1, 16)
        oc = o.contacts()
        assert np.array_equal(gc[:, 13:], oc[:, 13:]), "contact geom ids / dims differ"
        # MPR pairs (cylinder / capsule / mesh vs box ...) stop at opt.mpr_tolerance = 1e-6: rounding differences move such a contact
        # by up to ~1e-8 (measured 3e-9), analytic pairs agree at 1e-12
        assert np.abs(gc[:, :13] - oc[:, :13]).max(initial=0.0) < 1e-7
        for field in ("qacc", "qfrc_constraint"):
            g, r = engine_b.debug_forward(env, field), o.field(field)
            scale = max(1.0, float(np.abs(r).max()))
            assert np.abs(g - r).max() <= 1e-6 * scale, (field, env, np.abs(g - r).max(), scale)
        o.close()
    assert (engine_b.status().cpu().numpy() == 0).all()


def test_scene_b_trajectory_parity(scene_b, engine_b, settled_b):
    """60 PID + mj_step sub-steps through the impact phase (30-40 condim-6 contacts, object-object coupling)"""
    blob, A, _ = scene_b
    qpos, qvel = settled_b[400]
    engine_b.set_state(qpos, qvel)
    tgt = np.tile(HOME + np.array([0.2, 0.1, -0.1, 0.1, 0.1, 0.3, -0.1]), (2, 1))
    engine_b.move_group("All", tgt, 1e-7, 60)
    assert engine_b.run() == 0
    gq, gv = engine_b.get_state()
    gq, gv = gq.cpu().numpy(), gv.cpu().numpy()
    assert (engine_b.status().cpu().numpy() == 0).all()
    for env in range(2):
        o = _oracle(blob)
        o.reset(qpos[env], qvel[env])
        r, s = o.move_group("All", tgt[env], 1e-7, 60)
        assert (r, s) == (2, 61)
        assert np.abs(gq[env] - o.qpos).max() < 1e-6, (env, np.abs(gq[env] - o.qpos).max())
        assert np.abs(gv[env] - o.qvel).max() < 1e-4
        o.close()


def test_scene_b_render_parity(scene_b, engine_b, settled_b):
    """capsules and cylinders in the ray caster: depth within 1e-4 m on >= 99.9 % of the pixels (silhouette pixels may flip)"""
    blob, A, _ = scene_b
    qpos, qvel = settled_b[400]
    engine_b.set_state(qpos, qvel)
    cam = int(np.asarray(A["cam_top_down"]).ravel()[0])
    rgb, depth = engine_b.render(cam, 200, 200)
    o = _oracle(blob)
    o.reset(qpos[0], qvel[0])
    orgb, odepth = o.render(cam, 200, 200)
    o.close()
    d = depth[0].cpu().numpy()
    assert 0.4 < float(d.min()) < 1.2  # objects between the camera (z = 2) and the table
    close = np.abs(d - odepth) < 1e-4
    assert close.mean() >= 0.999, close.mean()
    assert (np.abs(rgb[0].cpu().numpy().astype(int) - orgb.astype(int)).max(axis=2)[close] <= 1).mean() >= 0.999


def test_batched_env_scene_b_reset_and_step():
    """BatchedGraspEnv on the reference's default scene: reset (1 s settle), observe, one scripted grasp attempt per env"""
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    env = BatchedGraspEnv(4, scene="B")
    obs = env.reset()
    assert obs["depth"].shape == (4, 200, 200)
    d = obs["depth"].cpu().numpy()
    assert (d.min(axis=(1, 2)) > 0.7).all() and (d.min(axis=(1, 2)) < 1.15).all()  # objects on the table below the camera
    rng = np.random.RandomState(0)
    obs, reward, done, info = env.step(env.sample_actions(rng))
    assert reward.shape == (4,) and set(np.unique(reward)) <= {0, 1}
    assert env.total_substeps() > 4 * 500
    assert (env.engine.status().cpu().numpy() == 0).all()  # no contact-list overflow
    env.close()


def test_cta_per_env_build_matches_warp_per_env_build(scene_a):
    """the same scene-A trajectory through both builds of the engine: warp-per-env, and (GE_CTA_PER_ENV=1) the big-scene build,
    a CTA of 4 warps per env.  Same arithmetic per item; the reductions over dofs / contacts
    are summed in a different (each fixed) order, so the two agree to rounding, not bit for bit."""
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, A, _ = scene_a
    qpos = np.stack([reset_qpos_scene_a(A, i) for i in range(4)])
    tgt = np.tile(HOME + np.array([0.3, 0.2, -0.2, 0.1, 0.1, 0.5, -0.1]), (4, 1))
    res = []
    for flag in ("0", "1"):
        os.environ["GE_CTA_PER_ENV"] = flag
        try:
            eng = BatchedEngine(blob, 4, 0)
        finally:
            del os.environ["GE_CTA_PER_ENV"]
        assert eng.size(9) == int(flag)
        eng.set_state(qpos)
        eng.move_group("All", tgt, 1e-7, 200)
        assert eng.run() == 0
        q, v = eng.get_state()
        res.append((q.cpu().numpy().copy(), v.cpu().numpy().copy()))
        eng.close()
    assert np.abs(res[0][0] - res[1][0]).max() < 1e-9 and np.abs(res[0][1] - res[1][1]).max() < 1e-7


def test_facade_opens_reference_default_scene():
    """GraspEnv(file=<the reference's default MJCF>) = scene B behind the reference API: reset() (global numpy RNG, 1 s settle),
    observation shapes, one step() with a pixel action"""
    from mujoco_rl_ur5_b200.grasp_env import GraspEnv

    np.random.seed(3)
    env = GraspEnv(file="/UR5+gripper/UR5gripper_2_finger_many_objects.xml", quiet=True, show_obs=False)
    assert env.scene == "B" and env.engine.size(9) == 1
    obs = env.reset()
    assert obs["rgb"].shape == (200, 200, 3) and obs["depth"].shape == (200, 200)
    assert 0.7 < float(np.min(obs["depth"])) < 1.15
    q = env.engine.get_state()[0][0].cpu().numpy()
    z = q[10:288:7]
    assert (z < 1.2).all() and (z > -0.1).all()  # every object has landed (table, or the floor next to it)
    obs, reward, done, info = env.step([100 * 200 + 100, 2])
    assert reward in (0, 1) and done is False
    env.close()


def test_scene_b_grasp_attempt_parity(scene_b):
    """a whole move_and_grasp attempt into the 40-object pile (~1900 sub-steps): reward bit-exact, all per-phase step counts equal,
    arm joint angles within the north-star tolerance 1e-4.  Individual objects of a pile may end up displaced (measured: one object
    by 2 cm, every other coordinate < 1e-6): contact dynamics between many bodies amplify rounding differences."""
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, A, _ = scene_b
    o = _oracle(blob)
    o.reset(reset_qpos_scene_b(A, 0))
    o.move_group("All", HOME + np.array([0, 0, 0, 0, 0, 0, 0.001]), 1e-9, 499)
    q, v = o.qpos.copy(), o.qvel.copy()
    pos = q[8:288].reshape(40, 7)[:, :3]
    on_table = (pos[:, 2] > 0.85) & (pos[:, 2] < 1.0)
    k = int((np.linalg.norm(pos[:, :2] - np.array([0.0, -0.6]), axis=1) + (~on_table) * 10).argmin())
    coords = np.array([pos[k, 0], pos[k, 1], pos[k, 2] + 0.02])
    eng = BatchedEngine(blob, 1, 0)
    eng.set_state(q[None], v[None])
    eng.grasp(coords[None], np.array([1], dtype=np.int32), 0.91)
    assert eng.run() == 0
    _, _, reward, _ = eng.results()
    info = eng.grasp_info().cpu().numpy()[0].tolist()
    gq = eng.get_state()[0][0].cpu().numpy()
    assert int(eng.status()[0]) == 0
    eng.close()
    o.reset(q, v)
    r, oinfo = o.move_and_grasp(coords, 1, 0.91)
    assert int(reward[0]) == r and info == oinfo, (int(reward[0]), r, info, oinfo)
    assert np.abs(gq[:8] - o.qpos[:8]).max() < 1e-4
    assert np.median(np.abs(gq - o.qpos)) < 1e-6
    o.close()


@pytest.mark.xfail(strict=False, reason="open defect of the CTA-per-env build (DESIGN.md section 4, r02k-r02q): whole grasp attempts of 1024 scene-B "
                   "environments with the action set bench.py drew in r02k end in an illegal memory access inside k_run (index arrays of the int "
                   "workspace overwritten); five other action sets run clean.  Runs in a child process: a CUDA fault must not poison this one.")
def test_whole_grasp_attempts_at_1024_envs_known_action_set():
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "repro_config5.py"), "1024", "1", "0", "bench"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-500:], [l for l in r.stderr.splitlines() if "rror" in l][-3:])
    assert "flagged envs 0" in r.stdout, r.stdout[-500:]
