"""Residency of the scene-A sub-step kernel: ten environments per SM, and the Hessian overflow row of the warp-per-env build.

The warp-per-env workspace is laid out by lifetime and its Newton Hessian region is capped so that ten warps share an SM (one CTA
of ten warps on the H100, which also grants the registers for it); a Hessian build whose blocks do not fit the region runs in the env's HBM overflow row with the same arithmetic in the same order.
So the results must not depend on the cap: the re-synchronised replay of tests/golden/replay_256.json (16 envs x 16 grasp attempts)
is run at the default cap and at the smallest cap GE_HCAP accepts, each in a child process (GE_HCAP is read at ge_create), and
every output is compared bit for bit.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "replay_256.json")
SMEM_PER_CTA = 232448  # H100: at most 227 KB of shared memory per CTA (228 KB per SM, 1 KB reserved per resident CTA)

_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv
g = json.load(open(sys.argv[2]))
st = np.load(sys.argv[2].replace(".json", "_states.npz"))
n, T = g["n_envs"], g["n_steps"]
env = BatchedGraspEnv(n, "A", 0, seed_base=20000, settle_ms=1000)
out = {k: [] for k in ("qpos", "qvel", "reward", "executed", "ginfo")}
for k in range(T):
    env.engine.set_state(st["qpos0"][:, k], st["qvel0"][:, k])
    env.current_observation = None
    actions = np.array([g["envs"][i][k]["action"] for i in range(n)], dtype=np.int32)
    obs, reward, done, info = env.step(actions)
    qpos, qvel = env.engine.get_state()
    out["qpos"].append(qpos.cpu().numpy()); out["qvel"].append(qvel.cpu().numpy())
    out["reward"].append(np.asarray(reward))
    out["executed"].append(info["executed"].cpu().numpy()); out["ginfo"].append(env.engine.grasp_info().cpu().numpy())
np.savez(sys.argv[3], **{k: np.stack(v) for k, v in out.items()})
print(json.dumps({"hcap": env.engine.size(10), "hfull": env.engine.size(11), "overflow_builds": env.engine.size(13)}))
env.close()
"""


def _replay(tmp, hcap=None):
    envv = dict(os.environ)
    envv.pop("GE_HCAP", None)
    if hcap is not None:
        envv["GE_HCAP"] = str(hcap)
    out = os.path.join(tmp, "replay_%s.npz" % (hcap or "default"))
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, GOLD, out], env=envv, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1]), dict(np.load(out))


@pytest.mark.gpu
def test_scene_a_workspace_fits_ten_envs_per_sm(scene_a):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, _, _ = scene_a
    eng = BatchedEngine(blob, 64, 0)
    ws, wpb, hcap, hfull, per_sm = (eng.size(k) for k in (7, 8, 10, 11, 12))
    maxcon, nbody = eng.size(6), eng.size(2)
    print(f"scene A: workspace {ws} B per env, {wpb} envs per CTA, Hessian region {hcap} of {hfull} doubles, {per_sm} envs per SM")
    assert eng.size(9) == 0  # warp-per-env build
    assert wpb == 10
    assert wpb * ws <= SMEM_PER_CTA
    assert per_sm == 10  # what the occupancy API grants with the kernel's registers and static shared memory
    assert 6 * maxcon + 6 * nbody <= hcap < hfull
    eng.close()


@pytest.mark.gpu
def test_replay_at_minimum_hessian_region_equals_default_bit_for_bit(scene_a):
    _, arrays, _ = scene_a
    tdn = np.asarray(arrays["tree_dofnum"])
    nbody = int(np.asarray(arrays["nbody"]).reshape(-1)[0])
    need_min = max(int((tdn * (tdn + 1) // 2).sum()), 6 * 32 + 6 * nbody)  # 32 contacts per env in scene A
    tmp = tempfile.mkdtemp()
    info_lo, lo = _replay(tmp, need_min)
    info_hi, hi = _replay(tmp)
    print("minimum region:", info_lo, "default region:", info_hi)
    assert info_lo["hcap"] == need_min and info_hi["hcap"] > need_min
    for k in hi:
        assert lo[k].shape == hi[k].shape and np.array_equal(lo[k], hi[k]), k
    assert info_lo["overflow_builds"] > 0  # the replay does reach the overflow row
    assert info_lo["overflow_builds"] >= info_hi["overflow_builds"]
