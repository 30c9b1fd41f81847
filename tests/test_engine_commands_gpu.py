"""The engine's command layer over a batch, against the fp64 oracle: env masks, mixed movement outcomes in one ge_run, partial runs and
busy accounting, gains, targets, controls and open-loop steps, in the warp-per-env build (scene A) and the CTA-per-env build (scene B).

Per-env controller state lives in EnvArrays and is written by small kernels of csrc/grasp_engine.cu (k_set_state, k_set_gain, k_command,
k_targets, k_ctrl, k_step_open, k_busy / k_count_busy); k_run hands one movement over to the next.  Every env here has its own OracleEnv,
reset to the same state and replaying the commands that env was given.

An env outside a mask must be untouched: qpos, qvel, targets, controls, results (result, steps, reward, total sub-steps), grasp info,
status, busy and the warm start (seen through debug_forward(env, "qacc"), which starts the solver from it) bit for bit, after the masked
call and after the next ge_run.

Step accounting, as the oracle's move_group loop runs it: a movement starts at step count 1, and each check evaluates the PID, tests
the tolerance, then ends with result 2 if the count is above max_steps, else takes one sub-step and counts it.  So max_steps = M ends
with result 2 after M + 1 counts and M sub-steps, and k_run needs M + 1 iterations for it (the closing check has no sub-step); a
movement that reaches its tolerance ends with result 1 after its sub-step, in as many iterations as sub-steps.  Inside a program (stay,
grasp) the closing check of one movement and the first sub-step of the next share an iteration.

Tolerances as tests/test_parity_gpu.py gates them: counts, results, rewards, grasp info and status exact; qpos 1e-6 and qvel 1e-4 over a
few hundred sub-steps; the arm within 1e-4 over a whole grasp attempt; bare open-loop sub-steps qpos 1e-9 and qvel 1e-7; the last PID
outputs within 1e-9 x their scale and targets (copies, or the IK solution of move_ee) within 1e-12.
"""
import json
import os

import numpy as np
import pytest

from tests.common import HOME

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ARM, GRIPPER, ALL = 0x1F, 0x40, 0x7F
SNAP_KEYS = ("qpos", "qvel", "target", "ctrl", "result", "steps", "reward", "total", "info", "status", "busy", "qacc")


@pytest.fixture(scope="module")
def success():
    """settled scene-A states (qpos0, qvel0) and the oracle's grasp attempt from each (records: coords, action, reward, info)"""
    z = np.load(os.path.join(GOLDEN, "success_64.npz"))
    recs = json.load(open(os.path.join(GOLDEN, "success_64.json")))["records"]
    return z["qpos0"], z["qvel0"], recs


def _oracle(blob):
    from oracle.oracle_py import OracleEnv

    return OracleEnv(blob)


def _engine(blob, n):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    return BatchedEngine(blob, n, 0)


def _mask(n, envs):
    m = np.zeros(n, np.uint8)
    m[list(envs)] = 1
    return m


def _snap(eng):
    """everything a masked call must leave alone, per env, on the host"""
    qpos, qvel = eng.get_state()
    result, steps, reward, total = eng.results()
    s = {"qpos": qpos, "qvel": qvel, "target": eng.get_targets(), "ctrl": eng.get_ctrl(), "result": result, "steps": steps,
         "reward": reward, "total": total, "info": eng.grasp_info(), "status": eng.status(), "busy": eng.busy()}
    s = {k: v.cpu().numpy() for k, v in s.items()}
    s["qacc"] = np.stack([eng.debug_forward(e, "qacc") for e in range(eng.n_envs)])
    return s


def _assert_untouched(before, after, envs, what):
    for e in envs:
        for k in SNAP_KEYS:
            assert before[k][e].tobytes() == after[k][e].tobytes(), (what, "env", e, k, before[k][e], after[k][e])


def _assert_same(a, b, ea, eb, what, keys=SNAP_KEYS):
    """env ea of snapshot a bit-identical to env eb of snapshot b"""
    for k in keys:
        assert a[k][ea].tobytes() == b[k][eb].tobytes(), (what, ea, eb, k, a[k][ea], b[k][eb])


class Ref:
    """one oracle env replaying the commands one engine env was given; result and step count as ge_get_results reports them, and the
    k_run iterations the last command takes (see the module docstring)"""

    def __init__(self, blob, qpos, qvel=None):
        self.o = _oracle(blob)
        self.o.reset(qpos, qvel)
        self.sub0 = self.o.substeps
        self.result = self.steps = self.reward = 0
        self.info = [0] * 12
        self.iters = 0

    def _ended(self, r, s):
        self.result, self.steps, self.iters = r, s, s - 1 + (r == 2)

    def group(self, mask, target, tol, max_steps):
        """target: the values of the group's members, or None"""
        self._ended(*self.o.move_group(mask, target, tol, max_steps))

    def ee(self, xyz, tol, max_steps):
        r, s = self.o.move_ee(np.asarray(xyz, np.float64), tol, max_steps)
        if r == 0:
            self.result, self.steps, self.iters = 3, 0, 0
        else:
            self._ended(r, s)

    def stay(self, ms):
        """orc_stay's chunks one by one (test_oracle_stay_is_chunks_of_ten_substeps pins that they are orc_stay); no chunk leaves the
        previous result and step count"""
        sub, self.iters = 0, 0
        for _ in range((ms // 2 + 9) // 10):
            r, s = self.o.move_group(ALL, None, 1e-7, 10)
            self.result, self.steps = r, s
            sub += s - 1
            self.iters = sub + (r == 2)

    def grasp(self, coords, rot, table=0.91):
        self.reward, self.info = self.o.move_and_grasp(np.asarray(coords, np.float64), int(rot), table)

    @property
    def substeps(self):
        return self.o.substeps - self.sub0

    def close(self):
        self.o.close()


def _check(g, g0, e, ref, what, qtol=1e-6, vtol=1e-4, counts=True, arm_only=False):
    """env e of snapshot g (taken after the commands; g0 before them) against its oracle"""
    o = ref.o
    if counts:
        assert (int(g["result"][e]), int(g["steps"][e])) == (ref.result, ref.steps), (what, e, g["result"][e], g["steps"][e], ref.result, ref.steps)
    assert int(g["total"][e] - g0["total"][e]) == ref.substeps, (what, e, int(g["total"][e] - g0["total"][e]), ref.substeps)
    assert int(g["reward"][e]) == ref.reward and g["info"][e].tolist() == list(ref.info), (what, e, g["reward"][e], g["info"][e], ref.reward, ref.info)
    assert int(g["status"][e]) == 0 and int(g["busy"][e]) == 0, (what, e, g["status"][e], g["busy"][e])
    n = 8 if arm_only else len(o.qpos)
    dq = np.abs(g["qpos"][e][:n] - o.qpos[:n]).max()
    assert dq < qtol, (what, e, "qpos", dq)
    if not arm_only:
        dv = np.abs(g["qvel"][e] - o.qvel).max()
        assert dv < vtol, (what, e, "qvel", dv)
        dc = np.abs(g["ctrl"][e] - o.ctrl).max()
        assert dc <= 1e-9 * max(1.0, float(np.abs(o.ctrl).max())), (what, e, "ctrl", dc, g["ctrl"][e], o.ctrl)
    dt = np.abs(g["target"][e] - o.target).max()
    assert dt <= 1e-12, (what, e, "target", dt, g["target"][e], o.target)


# ---------------------------------------------------------------------------------------------------------------- CPU: the oracle's side
def test_oracle_counting_edges(scene_a, success):
    """orc_move_group: max_steps 0 -> (2, 1) and no sub-step; tolerance reached at the first check -> (1, 2) and one sub-step;
    max_steps 1 -> (2, 2) and one sub-step; every check refreshes ctrl and last_input, a sub-step follows every check but the closing one"""
    blob, A, _ = scene_a
    qpos, qvel, _ = success
    adr = np.asarray(A["jnt_qposadr"]).ravel()[np.asarray(A["actuator_jntid"]).ravel()]
    far = qpos[0][:5] + [0.5, 0, 0, 0, 0]
    o = _oracle(blob)
    for target, tol, ms, want in ((far, 1e-12, 0, (2, 1, 0)), (None, 1e9, 50, (1, 2, 1)), (far, 1e-12, 1, (2, 2, 1)), (far, 1e-12, 7, (2, 8, 7))):
        o.reset(qpos[0], qvel[0])
        s0 = o.substeps
        r, s = o.move_group("Arm", target, tol, ms)
        assert (r, s, o.substeps - s0) == want, (target is None, tol, ms, r, s, o.substeps - s0)
        # the closing check of a max-steps movement evaluates the PID on the final joint angles; a tolerance end steps after it
        assert np.array_equal(o.last_input, o.qpos[adr]) == (r == 2), (tol, ms)
    o.close()


def test_oracle_stay_is_chunks_of_ten_substeps(scene_a, success):
    """orc_stay(ms) = ceil(ms / 2 / 10) movements of the whole robot to its targets, 10 sub-steps at most each (tolerance 1e-7): with
    the targets away from the joints every chunk runs its 10; and a held pose ends the first chunk after one sub-step"""
    blob = scene_a[0]
    qpos, qvel, _ = success
    o, p = _oracle(blob), _oracle(blob)
    for ms, chunks in ((0, 0), (1, 0), (2, 1), (19, 1), (20, 1), (21, 1), (22, 2), (41, 2), (42, 3), (100, 5)):
        for far in (True, False):
            for x in (o, p):
                x.reset(qpos[0], qvel[0])
                if far:
                    x.target[:5] += 0.3
            s0 = o.substeps
            o.stay(ms)
            n = 0
            for _ in range(chunks):
                r, s = p.move_group(ALL, None, 1e-7, 10)
                n += s - 1
                assert (r, s) == (2, 11) or not far, (ms, r, s)
            assert o.substeps - s0 == n and (not far or n == 10 * chunks), (ms, far, o.substeps - s0, n)
            assert np.array_equal(o.qpos, p.qpos) and np.array_equal(o.ctrl, p.ctrl) and np.array_equal(o.last_input, p.last_input)
    o.reset(qpos[0], qvel[0])
    s0 = o.substeps
    o.stay(20)
    assert o.substeps - s0 == 1, "a held pose reaches the 1e-7 tolerance at the first check"
    o.close()
    p.close()


def test_oracle_reset_and_open_loop_step(scene_a, success):
    """orc_reset restores the default gains, zeroes ctrl and sets target = last_input = the actuated joint angles, qacc warm start 0;
    orc_step uses ctrl clamped to actuator_ctrlrange but leaves ctrl raw, and leaves last_input, target and kp alone"""
    blob, A, _ = scene_a
    qpos, qvel, _ = success
    kp0 = np.asarray(A["pid_kp"], np.float64).ravel()
    rng = np.asarray(A["actuator_ctrlrange"], np.float64).reshape(-1, 2)
    adr = np.asarray(A["jnt_qposadr"]).ravel()[np.asarray(A["actuator_jntid"]).ravel()]
    o = _oracle(blob)
    o.reset(qpos[1], qvel[1])
    o.move_group("Arm", qpos[1][:5] + 0.2, 1e-12, 5)
    o.kp[:] = 3.0
    o.ctrl[:] = 9.0
    o.target[:] = -9.0
    o.last_input[:] = 7.0
    o.reset(qpos[0], qvel[0])
    assert np.array_equal(o.kp, kp0) and not o.ctrl.any() and not o.qacc_warmstart.any()
    assert np.array_equal(o.target, qpos[0][adr]) and np.array_equal(o.last_input, qpos[0][adr])
    assert np.array_equal(o.qpos, qpos[0]) and np.array_equal(o.qvel, qvel[0])
    o.reset(qpos[0])
    assert not o.qvel.any()
    raw = np.where(np.arange(7) % 2 == 0, 2.5, -1.75) * rng[:, 1]  # beyond the range on both sides
    clipped = np.clip(raw, rng[:, 0], rng[:, 1])
    states = []
    for c in (raw, clipped):
        o.reset(qpos[0], qvel[0])
        tg, li = o.target.copy(), o.last_input.copy()
        o.ctrl[:] = c
        o.step(5)
        assert np.array_equal(o.ctrl, c), "orc_step keeps the raw controls"
        assert np.array_equal(o.last_input, li) and np.array_equal(o.target, tg) and np.array_equal(o.kp, kp0)
        states.append((o.qpos.copy(), o.qvel.copy()))
    assert np.array_equal(states[0][0], states[1][0]) and np.array_equal(states[0][1], states[1][1]), "the step clamps to ctrlrange"
    o.close()


# ---------------------------------------------------------------------------------------------------------------- GPU: scene A
N = 16


@pytest.mark.gpu
@pytest.mark.parametrize("with_qvel", [True, False])
def test_masked_set_state(scene_a, success, with_qvel):
    """set_state under a mask on envs that have moved, with per-env gains and raw controls: the selected envs get the new state, zero or
    given qvel, targets = the actuated joint angles, ctrl 0, results / info / status cleared and the default gains (a follow-up movement
    matches an oracle that was only reset); the others are untouched and keep their gains"""
    blob, A, _ = scene_a
    qpos, qvel, _ = success
    kp0 = np.asarray(A["pid_kp"], np.float64).ravel()
    adr = np.asarray(A["jnt_qposadr"]).ravel()[np.asarray(A["actuator_jntid"]).ravel()]
    eng = _engine(blob, N)
    sel = [0, 3, 7, 8, 12, N - 1]
    rest = [e for e in range(N) if e not in sel]
    kpv = {0: kp0[0] * (0.5 + np.arange(N) / N), 2: kp0[2] * (1.5 - np.arange(N) / (2 * N))}
    tg1 = qpos[:N, :5] + [0.2, -0.1, 0.1, 0.05, -0.05]
    ctrl = np.linspace(-0.9, 0.9, N * 7).reshape(N, 7)
    eng.set_state(qpos[:N], qvel[:N])
    for a, v in kpv.items():
        eng.set_gain(a, v)
    eng.move_group("Arm", tg1, 1e-12, 20)
    assert eng.run() == 0
    eng.set_ctrl(ctrl)
    before = _snap(eng)
    new_q, new_v = qpos[N:2 * N], qvel[N:2 * N]
    eng.set_state(new_q, new_v if with_qvel else None, env_mask=_mask(N, sel))
    after = _snap(eng)
    _assert_untouched(before, after, rest, "set_state")
    for e in sel:
        assert np.array_equal(after["qpos"][e], new_q[e]) and np.array_equal(after["qvel"][e], new_v[e] if with_qvel else np.zeros_like(new_v[e]))
        assert np.array_equal(after["target"][e], new_q[e][adr]) and not after["ctrl"][e].any()
        assert (after["result"][e], after["steps"][e], after["reward"][e], after["status"][e], after["busy"][e]) == (0, 0, 0, 0, 0)
        assert not after["info"][e].any() and after["total"][e] == before["total"][e]
    # follow-up movement of every env: default gains where the state was set, the custom ones elsewhere
    tg2 = HOME[:5] + [0.1, 0.05, -0.05, 0.0, 0.1]
    eng.move_group("Arm", np.tile(tg2, (N, 1)), 0.01, 60)
    assert eng.run() == 0
    g = _snap(eng)
    for e in range(N):
        if e in sel:
            ref = Ref(blob, new_q[e], new_v[e] if with_qvel else None)
        else:
            ref = Ref(blob, qpos[e], qvel[e])
            for a, v in kpv.items():
                ref.o.kp[a] = v[e]
            ref.group(ARM, tg1[e], 1e-12, 20)
            ref.o.ctrl[:] = ctrl[e]
        ref.sub0 = ref.o.substeps  # `after` holds the totals from here
        ref.group(ARM, tg2, 0.01, 60)
        _check(g, after, e, ref, ("follow-up", e in sel))
        ref.close()
    # the custom gains matter: with the default ones the follow-up of an unselected env is far from the engine's
    o = Ref(blob, qpos[rest[0]], qvel[rest[0]])
    o.group(ARM, tg1[rest[0]], 1e-12, 20)
    o.group(ARM, tg2, 0.01, 60)
    assert np.abs(o.o.qpos[:5] - g["qpos"][rest[0]][:5]).max() > 1e-4
    o.close()
    eng.close()


def _mixed_batch(qpos):
    """(role, command) per env of the mixed batch; the commands of one role go out in one masked call"""
    arm = qpos[:, :5]
    far = arm + [0.5, 0, 0, 0, 0]
    return [
        ("success", ("group", ARM, arm + [0.15, -0.1, 0.1, 0.1, -0.1], 0.05, 400)),
        ("idle", None),
        ("max_steps", ("group", GRIPPER, np.full((len(qpos), 1), -0.4), 0.01, 60)),
        ("custom_mask", ("group", 0b1000101, np.stack([arm[:, 0] - 0.1, arm[:, 2] + 0.1, np.full(len(qpos), 0.1)], 1), 0.02, 300)),
        ("idle", None),
        ("ee", ("ee", np.tile([0.1, -0.5, 1.0], (len(qpos), 1)), 0.05, 400)),
        ("ee_unreachable", ("ee", np.tile([5.0, 5.0, 5.0], (len(qpos), 1)), 0.05, 400)),
        ("stay1", ("stay", 1)),
        ("idle", None),
        ("stay20", ("stay", 20)),
        ("stay22", ("stay", 22)),
        ("max_steps_0", ("group", ARM, far, 1e-12, 0)),
        ("idle", None),
        ("tol_first_check", ("group", ARM, None, 1e9, 50)),
        ("max_steps_1", ("group", ARM, far, 1e-12, 1)),
        ("idle", None),
    ]


def _issue(eng, batch, envs=None):
    """send each role's command to its envs (among `envs`) through a mask"""
    n = eng.n_envs
    envs = range(n) if envs is None else envs
    for e, (role, cmd) in enumerate(batch):
        if cmd is None or e not in envs:
            continue
        m = _mask(n, [e])
        if cmd[0] == "group":
            eng.move_group(cmd[1], cmd[2], cmd[3], cmd[4], env_mask=m)
        elif cmd[0] == "ee":
            eng.move_ee(cmd[1], cmd[2], cmd[3], env_mask=m)
        else:
            eng.stay(cmd[1], env_mask=m)


def _replay(ref, cmd, e):
    if cmd is None:
        return
    if cmd[0] == "group":
        ref.group(cmd[1], None if cmd[2] is None else cmd[2][e], cmd[3], cmd[4])
    elif cmd[0] == "ee":
        ref.ee(cmd[1][e], cmd[2], cmd[3])
    else:
        ref.stay(cmd[1])


EXPECT = {"success": (1, None, None), "custom_mask": (1, None, None), "ee": (1, None, None), "max_steps": (2, 61, 60), "ee_unreachable": (3, 0, 0), "stay1": (0, 0, 0), "stay20": (1, 2, 1),
          "stay22": (2, 11, 11), "max_steps_0": (2, 1, 0), "tol_first_check": (1, 2, 1), "max_steps_1": (2, 2, 1), "idle": (0, 0, 0)}


@pytest.mark.gpu
def test_mixed_outcomes_in_one_run(scene_a, success):
    """success, max-steps, a custom group with a partial target, move_ee reachable and not, stay(1 / 20 / 22), the counting edges and
    idle envs in ONE ge_run: each env matches its oracle; envs without a command are untouched"""
    blob = scene_a[0]
    qpos, qvel, _ = success
    eng = _engine(blob, N)
    batch = _mixed_batch(qpos[:N])
    eng.set_state(qpos[:N], qvel[:N])
    g0 = _snap(eng)
    _issue(eng, batch)
    issued = _snap(eng)
    unmoved = [e for e, (r, _) in enumerate(batch) if r in ("idle", "stay1")]
    failed = [e for e, (r, _) in enumerate(batch) if r == "ee_unreachable"]
    no_result = tuple(k for k in SNAP_KEYS if k != "result")
    _assert_untouched(g0, issued, unmoved, "issued")
    for e in failed:  # a failed IK reports result 3 at once and touches nothing else
        assert issued["result"][e] == 3
        _assert_same(g0, issued, e, e, "failed move_ee", keys=no_result)
    assert eng.run() == 0
    g = _snap(eng)
    _assert_untouched(g0, g, unmoved, "run")
    for e in failed:
        _assert_same(g0, g, e, e, "failed move_ee, run", keys=no_result)
    for e, (role, cmd) in enumerate(batch):
        ref = Ref(blob, qpos[e], qvel[e])
        _replay(ref, cmd, e)
        r, s, sub = EXPECT[role] if role in EXPECT else (ref.result, ref.steps, ref.substeps)
        # the oracle gives each role the outcome it stands for
        assert ref.result == r and (s is None or ref.steps == s) and (sub is None or ref.substeps == sub), (role, ref.result, ref.steps, ref.substeps)
        _check(g, g0, e, ref, role)
        ref.close()
    eng.close()


@pytest.mark.gpu
def test_partial_runs_and_busy_accounting(scene_a, success):
    """ge_run(max_substeps=K) just before, at and after movement ends (K = M and M + 1 for max_steps M = 60, around the end of the
    successful movement, around the counting edges): n_busy and ge_get_busy follow the iteration rule; a masked command to the idle envs
    then runs beside the unfinished ones, and every env matches the oracle of its command sequence"""
    blob = scene_a[0]
    qpos, qvel, _ = success
    eng = _engine(blob, N)
    batch = _mixed_batch(qpos[:N])
    refs = []
    for e, (role, cmd) in enumerate(batch):
        ref = Ref(blob, qpos[e], qvel[e])
        _replay(ref, cmd, e)
        refs.append((ref.o.qpos.copy(), ref.result, ref.steps, ref.iters))
        ref.close()
    iters = np.array([r[3] for r in refs])
    succ = iters[0]
    assert iters[2] == 61 and iters[11] == 1 and iters[13] == 1 and iters[14] == 2 and iters[10] == 12 and iters[9] == 1
    tg = HOME[:5] + [0.1, 0.0, 0.05, 0.0, 0.0]
    for K in sorted({1, 2, 11, 12, 60, 61, succ - 1, succ}):
        eng.set_state(qpos[:N], qvel[:N])
        g0 = _snap(eng)
        _issue(eng, batch)
        n_busy = eng.run(max_substeps=K)
        busy = eng.busy().cpu().numpy()
        want = (iters > K).astype(np.uint8)
        assert n_busy == int(want.sum()) and np.array_equal(busy, want), (K, n_busy, busy.tolist(), iters.tolist())
        mid = _snap(eng)
        idle = [e for e in range(N) if not want[e]]
        for e in idle:  # finished: the final result already
            assert (mid["result"][e], mid["steps"][e]) == refs[e][1:3], (K, e, mid["result"][e], mid["steps"][e], refs[e])
        eng.move_group("Arm", np.tile(tg, (N, 1)), 0.05, 80, env_mask=_mask(N, idle))
        assert eng.run() == 0
        g = _snap(eng)
        for e, (role, cmd) in enumerate(batch):
            ref = Ref(blob, qpos[e], qvel[e])
            _replay(ref, cmd, e)
            if e in idle:
                ref.group(ARM, tg, 0.05, 80)
            _check(g, g0, e, ref, (K, role))
            ref.close()
    eng.close()


@pytest.mark.gpu
def test_sparse_mask_is_batch_invariant(scene_a, success):
    """5 busy envs among 64 (two grasp attempts, three movements) end bit-identical to a 5-env engine given the same commands; the other
    59 are untouched"""
    blob = scene_a[0]
    qpos, qvel, recs = success
    n = 64
    sel = [0, 17, 40, 48, 63]
    grasp = {0: recs[0], 48: recs[48]}
    assert recs[0]["reward"] == 1 and recs[48]["reward"] == 0

    def drive(eng, envs):
        k = {e: i for i, e in enumerate(envs)}
        pick = lambda es: _mask(eng.n_envs, [k[e] for e in es])
        coords, rot = np.zeros((eng.n_envs, 3)), np.zeros(eng.n_envs, np.int32)
        for e, r in grasp.items():
            coords[k[e]], rot[k[e]] = r["coords"], r["action"][1]
        eng.grasp(coords, rot, 0.91, env_mask=pick(grasp))
        eng.move_group("Arm", np.tile(HOME[:5] + [0.2, -0.1, 0.1, 0.0, 0.1], (eng.n_envs, 1)), 0.01, 300, env_mask=pick([17]))
        eng.move_ee(np.tile([0.15, -0.55, 1.05], (eng.n_envs, 1)), 0.01, 500, env_mask=pick([40]))
        eng.stay(60, env_mask=pick([63]))
        assert eng.run() == 0

    big = _engine(blob, n)
    big.set_state(qpos[:n], qvel[:n])
    b0 = _snap(big)
    drive(big, list(range(n)))
    b = _snap(big)
    big.close()
    small = _engine(blob, len(sel))
    small.set_state(qpos[sel], qvel[sel])
    drive(small, sel)
    s = _snap(small)
    small.close()
    for i, e in enumerate(sel):
        _assert_same(b, s, e, i, "64 vs 5 envs")
    assert int(b["reward"][0]) == 1 and b["info"][0].tolist() == recs[0]["info"] and b["info"][48].tolist() == recs[48]["info"]
    _assert_untouched(b0, b, [e for e in range(n) if e not in sel], "unselected among 64")


@pytest.mark.gpu
def test_masked_grasp(scene_a, success):
    """grasp(..., env_mask) as BatchedGraspEnv.step issues it, in two rounds: executed envs match orc_move_and_grasp (reward and info
    exact, arm 1e-4); envs left out keep everything, their previous reward and info included"""
    blob = scene_a[0]
    qpos, qvel, recs = success
    rec = [0, 1, 2, 50, 51, 52, 3, 53]
    n = len(rec)
    eng = _engine(blob, n)
    eng.set_state(qpos[rec], qvel[rec])
    coords = np.array([recs[r]["coords"] for r in rec])
    rot = np.array([recs[r]["action"][1] for r in rec], np.int32)
    refs = [Ref(blob, qpos[r], qvel[r]) for r in rec]
    g0 = _snap(eng)
    prev = g0
    for rnd in ([0, 1, 3], [2, 4, 5, 6]):
        eng.grasp(coords, rot, 0.91, env_mask=_mask(n, rnd))
        assert eng.run() == 0
        g = _snap(eng)
        _assert_untouched(prev, g, [e for e in range(n) if e not in rnd], ("grasp round", rnd))
        for e in rnd:
            refs[e].grasp(coords[e], rot[e])
            _check(g, g0, e, refs[e], ("grasp", e), qtol=1e-4, counts=False, arm_only=True)
        prev = g
    assert sum(int(g["reward"][e]) for e in range(n)) >= 3 and int(g["reward"][0]) == 1  # rewarded attempts stay rewarded
    for r in refs:
        r.close()
    eng.close()


@pytest.mark.gpu
def test_targets_and_gains(scene_a, success):
    """set_targets / get_targets round-trip; move_group(target=None) drives to set targets; get_targets after move_ee holds the IK
    solution; set_gain with a scalar and with a per-env vector acts as o.kp[a]; a grasp attempt leaves kp[0] = 20 whatever it was"""
    blob = scene_a[0]
    qpos, qvel, recs = success
    n = 8
    eng = _engine(blob, n)
    eng.set_state(qpos[:n], qvel[:n])
    T = np.tile(HOME, (n, 1)) + np.linspace(-0.2, 0.2, n * 7).reshape(n, 7)
    eng.set_targets(T)
    assert eng.get_targets().cpu().numpy().tobytes() == T.tobytes()
    # gains: scalar on actuator 1, per-env vector on actuator 3
    kp3 = 5.0 + 4.0 * np.arange(n)
    eng.set_gain(1, 45.0)
    eng.set_gain(3, kp3)
    g0 = _snap(eng)
    m1 = [0, 2, 3, 6]
    eng.move_group("All", None, 0.05, 120, env_mask=_mask(n, m1))
    m2 = [1, 4, 7]
    xyz = np.tile([0.1, -0.5, 1.0], (n, 1)) + np.linspace(-0.05, 0.05, n)[:, None] * [1, 1, 0]
    eng.move_ee(xyz, 0.05, 150, env_mask=_mask(n, m2))
    tg = eng.get_targets().cpu().numpy()
    o = _oracle(blob)
    for e in range(n):
        if e in m2:
            o.reset(qpos[e], qvel[e])
            q5 = o.ik(xyz[e])
            assert q5 is not None and np.abs(tg[e][:5] - q5).max() <= 1e-12 and tg[e][5:].tobytes() == T[e][5:].tobytes(), (e, tg[e], q5)
        else:
            assert tg[e].tobytes() == T[e].tobytes()
    o.close()
    assert eng.run() == 0
    g = _snap(eng)
    for e in range(n):
        ref = Ref(blob, qpos[e], qvel[e])
        ref.o.target[:] = T[e]
        ref.o.kp[1], ref.o.kp[3] = 45.0, kp3[e]
        if e in m1:
            ref.group(ALL, None, 0.05, 120)
        elif e in m2:
            ref.ee(xyz[e], 0.05, 150)
        _check(g, g0, e, ref, ("targets and gains", e))
        ref.close()
    _assert_untouched(g0, g, [5], "no command")
    # kp[0] after a grasp attempt: 20 (GraspingEnv's 10 -> 20), from 33 and from 5; a follow-up movement of joint 0 shows it
    kp0 = {0: 33.0, 1: 5.0}
    eng.set_state(qpos[:n], qvel[:n])
    eng.set_gain(0, np.array([kp0.get(e, 21.0) for e in range(n)]))
    eng.grasp(np.array([recs[e]["coords"] for e in range(n)]), np.array([recs[e]["action"][1] for e in range(n)], np.int32), 0.91,
              env_mask=_mask(n, list(kp0)))
    assert eng.run() == 0
    g0 = _snap(eng)
    tg = g0["qpos"][:, :5] + [0.05, 0, 0, 0, 0]  # unsaturated: the PID output of joint 0 is proportional to kp[0]
    eng.move_group("Arm", tg, 1e-12, 40, env_mask=_mask(n, list(kp0)))
    assert eng.run() == 0
    g = _snap(eng)
    for e, kp in kp0.items():
        errs = []
        for keep in (False, True):  # the oracle's attempt ends with kp[0] = 20; `keep` puts the custom gain back
            ref = Ref(blob, qpos[e], qvel[e])
            ref.o.kp[0] = kp
            ref.grasp(recs[e]["coords"], recs[e]["action"][1])
            assert ref.o.kp[0] == 20.0
            assert int(g0["reward"][e]) == ref.reward and g0["info"][e].tolist() == ref.info, (e, g0["info"][e], ref.info)
            if keep:
                ref.o.kp[0] = kp
            ref.group(ARM, tg[e], 1e-12, 40)
            errs.append(np.abs(g["qpos"][e][:8] - ref.o.qpos[:8]).max())
            ref.close()
        assert (int(g["result"][e]), int(g["steps"][e])) == (2, 41)
        assert errs[0] < 1e-4 and errs[1] > 1e-3, (e, errs)
    eng.close()


@pytest.mark.gpu
def test_open_loop(scene_a, success):
    """set_ctrl under a mask with values beyond actuator_ctrlrange on both sides: get_ctrl returns them raw, the others keep theirs;
    step_open_loop(n, mask) for n = 1, 7, 40 matches o.ctrl[:] = ...; o.step(n) and adds n to total_substeps; envs left out are
    untouched.  One call of 48 sub-steps equals the three calls bit for bit (the qacc warm start is carried), clamped controls equal the
    raw ones bit for bit, and a closed-loop movement afterwards matches the oracle (the PID's last input is the one of set_state)"""
    blob, A, _ = scene_a
    qpos, qvel, _ = success
    rng = np.asarray(A["actuator_ctrlrange"], np.float64).reshape(-1, 2)
    rec = [0, 1, 2, 3, 4, 5, 0, 0]
    n = len(rec)
    eng = _engine(blob, n)
    eng.set_state(qpos[rec], qvel[rec])
    c0 = np.linspace(-0.5, 0.5, n * 7).reshape(n, 7) * rng[:, 1]
    eng.set_ctrl(c0)
    assert eng.get_ctrl().cpu().numpy().tobytes() == c0.tobytes()
    raw = np.array([2.5, -1.5, 3.0, -2.0, 1.5, -4.0, 1.25]) * rng[:, 1]  # every actuator beyond its range, both signs
    clipped = np.clip(raw, rng[:, 0], rng[:, 1])
    s1 = [0, 2, 5, 6]  # 6 has 0's state and controls; 7 has 0's state and the clamped controls
    c1 = np.full((n, 7), 9.0)  # rows outside the mask must not land
    c1[0] = c1[6] = raw
    # the gripper opens in every stepped env: closing it makes a contact within the 48 sub-steps, after which a 1e-14 nudge of the
    # state moves qvel by 2e-5 in the oracle itself, and no bare-step tolerance holds
    c1[2], c1[5] = -raw * [1, 1, 1, 1, 1, 1, -1], 0.8 * raw
    eng.set_ctrl(c1, env_mask=_mask(n, s1))
    c7 = np.full((n, 7), -9.0)
    c7[7] = clipped
    eng.set_ctrl(c7, env_mask=_mask(n, [7]))
    ctrl = c0.copy()
    ctrl[s1], ctrl[7] = c1[s1], clipped
    assert eng.get_ctrl().cpu().numpy().tobytes() == ctrl.tobytes()
    refs = {}
    for e in (0, 2, 3, 5):
        refs[e] = Ref(blob, qpos[rec[e]], qvel[rec[e]])
        refs[e].o.ctrl[:] = ctrl[e]
    s2 = sorted(refs)
    g0 = _snap(eng)
    prev = g0
    for k in (1, 7, 40):
        eng.step_open_loop(k, env_mask=_mask(n, s2))
        g = _snap(eng)
        _assert_untouched(prev, g, [e for e in range(n) if e not in s2], ("open loop", k))
        for e in s2:
            refs[e].o.step(k)
            assert g["total"][e] - prev["total"][e] == k
            assert g["ctrl"][e].tobytes() == ctrl[e].tobytes()
            dq, dv = np.abs(g["qpos"][e] - refs[e].o.qpos).max(), np.abs(g["qvel"][e] - refs[e].o.qvel).max()
            assert dq < 1e-9 and dv < 1e-7, (k, e, dq, dv)
            assert g["target"][e].tobytes() == prev["target"][e].tobytes()
        prev = g
    eng.step_open_loop(48, env_mask=_mask(n, [6, 7]))
    g = _snap(eng)
    _assert_untouched(prev, g, [e for e in range(n) if e not in (6, 7)], "open loop 48")
    _assert_same(g, g, 0, 6, "1 + 7 + 40 vs 48 sub-steps")
    _assert_same(g, g, 0, 7, "raw vs clamped controls", keys=("qpos", "qvel", "total", "status", "qacc"))
    # closed loop from here: the first PID evaluation differentiates against set_state's joint angles in both implementations
    tg = HOME[:5] + [0.1, -0.1, 0.1, 0.0, 0.0]
    eng.move_group("Arm", np.tile(tg, (n, 1)), 1e-12, 30, env_mask=_mask(n, s2))
    assert eng.run() == 0
    g2 = _snap(eng)
    _assert_untouched(g, g2, [1, 4, 6, 7], "closed loop")
    for e in s2:
        refs[e].group(ARM, tg, 1e-12, 30)
        _check(g2, g0, e, refs[e], ("closed loop after open loop", e))
        refs[e].close()
    eng.close()


@pytest.mark.gpu
def test_rejected_calls_change_nothing(scene_a, success):
    """bad arguments return GE_ERR_ARG and leave every env bit-identical, a pending movement included"""
    blob = scene_a[0]
    qpos, qvel, _ = success
    n = 4
    eng = _engine(blob, n)
    eng.set_state(qpos[:n], qvel[:n])
    eng.move_group("Arm", np.tile(HOME[:5] + 0.1, (n, 1)), 1e-12, 20, env_mask=_mask(n, [1, 2]))
    L, h = eng.L, eng.h
    GE_ERR_ARG = -1
    calls = [("ge_move_group 0", lambda: L.ge_move_group(h, 0, None, 0.1, 10, None)),
             ("ge_move_group 0x80", lambda: L.ge_move_group(h, 0x80, None, 0.1, 10, None)),
             ("ge_move_group -1", lambda: L.ge_move_group(h, -1, None, 0.1, 10, None)),
             ("ge_stay -1", lambda: L.ge_stay(h, -1, None)),
             ("ge_step_open_loop 0", lambda: L.ge_step_open_loop(h, 0, None)),
             ("ge_run_async 0", lambda: L.ge_run_async(h, 0)),
             ("ge_set_gain -1", lambda: L.ge_set_gain(h, -1, None, 5.0)),
             ("ge_set_gain 7", lambda: L.ge_set_gain(h, 7, None, 5.0)),
             ("ge_set_ctrl NULL", lambda: L.ge_set_ctrl(h, None, None))]
    before = _snap(eng)
    assert before["busy"].tolist() == [0, 1, 1, 0]
    for what, call in calls:
        assert call() == GE_ERR_ARG, what
        assert L.ge_last_error()
        after = _snap(eng)
        _assert_untouched(before, after, range(n), what)
    assert eng.run() == 0
    g = _snap(eng)
    for e in range(n):
        ref = Ref(blob, qpos[e], qvel[e])
        if e in (1, 2):
            ref.group(ARM, HOME[:5] + 0.1, 1e-12, 20)
        _check(g, before, e, ref, ("after rejected calls", e))
        ref.close()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- GPU: scene B
@pytest.mark.gpu
def test_scene_b_masked_open_loop_and_move(scene_b):
    """the CTA-per-env build: masked set_ctrl + step_open_loop and a short masked move_group from contact-heavy states, one of them with
    its Newton Hessian in the overflow row, against the oracle (the scene-B trajectory tolerances: qpos 1e-6, qvel 1e-4); envs left out
    are untouched"""
    blob, A, _ = scene_b
    z = np.load(os.path.join(GOLDEN, "scene_b_edges.npz"))
    states = [0, 3, 5, 2]  # 0 and 2: the two states whose Hessian blocks exceed the default region
    n = len(states)
    q, v = z["qpos"][states], z["qvel"][states]
    rng = np.asarray(A["actuator_ctrlrange"], np.float64).reshape(-1, 2)
    eng = _engine(blob, n)
    eng.set_state(q, v)
    assert int(eng.debug_forward(0, "hlayout")[0]) == 1, "state 0 builds its Newton Hessian in the overflow row"
    ctrl = np.array([1.5, -0.5, 1.25, -2.0, 0.5, 3.0, -1.5]) * rng[:, 1] * np.linspace(0.5, 1.0, n)[:, None]
    s1 = [0, 1, 2]
    eng.set_ctrl(ctrl, env_mask=_mask(n, s1))
    refs = {e: Ref(blob, q[e], v[e]) for e in range(n)}
    for e in s1:
        refs[e].o.ctrl[:] = ctrl[e]
    g0 = _snap(eng)
    assert g0["ctrl"][:3].tobytes() == ctrl[:3].tobytes() and not g0["ctrl"][3].any()
    prev = g0
    for k in (1, 7):
        eng.step_open_loop(k, env_mask=_mask(n, s1))
        g = _snap(eng)
        _assert_untouched(prev, g, [3], ("open loop", k))
        for e in s1:
            refs[e].o.step(k)
            assert g["total"][e] - prev["total"][e] == k and g["ctrl"][e].tobytes() == ctrl[e].tobytes()
            dq, dv = np.abs(g["qpos"][e] - refs[e].o.qpos).max(), np.abs(g["qvel"][e] - refs[e].o.qvel).max()
            assert dq < 1e-6 and dv < 1e-4, (k, e, dq, dv)
        prev = g
    s2 = [0, 2, 3]
    tg = HOME[:5] + [0.2, 0.0, 0.0, 0.0, 0.0]
    eng.move_group("Arm", np.tile(tg, (n, 1)), 1e-12, 6, env_mask=_mask(n, s2))
    assert eng.run() == 0
    g = _snap(eng)
    _assert_untouched(prev, g, [1], "move_group")
    for e in s2:
        refs[e].group(ARM, tg, 1e-12, 6)
        _check(g, g0, e, refs[e], ("scene B", e))
    for r in refs.values():
        r.close()
    eng.close()
