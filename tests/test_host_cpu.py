"""CPU tests of the host side: model blob, C-ABI surface, compat shims, sharding (world_size-2 gloo)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_blob_roundtrip_and_sizes(scene_a):
    from mujoco_rl_ur5_b200.model.blob import pack, unpack

    blob, A, names = scene_a
    assert [int(A[k][0]) for k in ("nbody", "njnt", "nq", "nv", "nu", "ngeom", "neq")] == [24, 32, 50, 44, 7, 36, 1]  # SURVEY 2.1
    again = unpack(pack(A))
    assert set(again) == set(A) and all(np.array_equal(again[k], A[k]) for k in A)
    assert names["body"][int(A["ee_body"][0])] == "ee_link" and names["camera"][int(A["cam_top_down"][0])] == "top_down"
    # actuated joints are joints 0..6 = qpos addresses 0..6 (MujocoController.py:43,319)
    assert list(A["actuator_jntid"]) == list(range(7)) and list(A["jnt_qposadr"][:8]) == list(range(8))
    # PID gains after p_scale=3, d_scale=0.1 (MujocoController.py:157-235)
    assert np.allclose(A["pid_kp"], [21, 30, 15, 21, 15, 15, 7.5]) and np.allclose(A["pid_kd"], [0.11, 0.1, 0.05, 0.01, 0.01, 0.01, 0])


@pytest.mark.skipif(not os.path.exists("/root/reference/UR5+gripper/UR5gripper_2_finger.xml"), reason="reference assets not present")
def test_compiler_reproduces_committed_blob():
    from mujoco_rl_ur5_b200.model.scene import compile_scene, load_scene

    for key in ("A", "A1"):  # A1: the 6-object scene with its objects turned into 4 cm cubes (BASELINE config 3)
        A, _ = load_scene(key)
        M = compile_scene(key)
        for k in ("body_mass", "body_inertia", "dof_invweight0", "pair_geom", "mesh_vert", "geom_obbhalf", "geom_size", "geom_type"):
            assert np.allclose(np.asarray(M[k]).reshape(A[k].shape), A[k], rtol=1e-12, atol=1e-14), (key, k)


def test_cabi_library_exports_every_declared_symbol():
    """libgrasp_engine.so loads without a GPU and exports exactly what include/grasp_engine.h declares (no compute calls here)."""
    from mujoco_rl_ur5_b200 import engine

    hdr = open(os.path.join(ROOT, "include", "grasp_engine.h")).read()
    declared = sorted(set(re.findall(r"\b(ge_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 25
    lib = ctypes.CDLL(engine.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in grasp_engine.h but not exported"
    assert set(engine.SYMBOLS) <= set(declared)
    lib.ge_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.ge_version()
    # argument validation does not need a device
    assert lib.ge_destroy(None) == 0
    h = ctypes.c_void_p()
    assert lib.ge_create(b"not a blob" * 8, 80, 4, 0, None, ctypes.byref(h)) < 0
    lib.ge_last_error.restype = ctypes.c_char_p
    assert b"blob" in lib.ge_last_error()


def test_create_refuses_a_tree_wider_than_a_lane_group(scene_a):
    """the mass solve gives every non-simple kinematic tree one 8-lane group: ge_create refuses a wider tree from the host blob,
    before any CUDA call, so the refusal needs no device"""
    from mujoco_rl_ur5_b200 import engine
    from mujoco_rl_ur5_b200.model.blob import pack, unpack

    arrays = unpack(scene_a[0])
    assert arrays["tree_dofnum"][0] == 8 and not arrays["tree_simple"][0]  # the arm
    arrays["tree_dofnum"][0] = 9
    blob = pack(arrays)
    lib = ctypes.CDLL(engine.LIB_PATH)
    lib.ge_last_error.restype = ctypes.c_char_p
    h = ctypes.c_void_p()
    assert lib.ge_create(blob, len(blob), 4, 0, None, ctypes.byref(h)) == -3  # GE_ERR_MODEL
    assert b"tree 0 has 9 dofs" in lib.ge_last_error()


def test_engine_refuses_to_run_without_gpu():
    """no CPU fallback: constructing the engine without CUDA must fail loudly"""
    import torch

    from mujoco_rl_ur5_b200.engine import BatchedEngine, EngineError
    from mujoco_rl_ur5_b200.model.scene import load_scene_blob

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(EngineError):
        BatchedEngine(load_scene_blob("A"), 2, 0)


def test_product_does_not_import_oracle():
    """only tests/, __graft_entry__.smoke() and bench.py may touch oracle/"""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "mujoco_rl_ur5_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                bad = re.search(r"^\s*(from|import)\s+oracle\b|#\s*include[^\n]*oracle|libgrasp_oracle|dlopen[^\n]*oracle", src, re.M)
                assert bad is None, (os.path.join(dirpath, f), bad.group(0))


def test_gym_shim_register_make_and_spaces():
    compat = os.path.join(ROOT, "mujoco_rl_ur5_b200", "compat")
    sys.path.insert(0, compat)
    try:
        import gym
        from gym import spaces
        from gym.envs.registration import register

        class Dummy:
            def __init__(self, a=1):
                self.a = a

        register(id="Dummy-v0", entry_point=Dummy)
        assert gym.make("Dummy-v0", a=5).a == 5
        md = spaces.MultiDiscrete([40000, 6])
        md.seed(0)
        s = md.sample()
        assert list(md.nvec) == [40000, 6] and 0 <= s[0] < 40000 and 0 <= s[1] < 6 and md.contains(s)
        from prettytable import PrettyTable
        from termcolor import colored

        t = PrettyTable(["Modules", "Parameters"])
        t.add_row(["conv", 12])
        assert "conv" in str(t) and "x" in colored("x", color="green", attrs=["bold"])
    finally:
        sys.path.remove(compat)
        for k in [k for k in sys.modules if k == "gym" or k.startswith("gym.") or k in ("termcolor", "prettytable")]:
            del sys.modules[k]


def test_shard_ranges_cover_and_seeds_are_global():
    from mujoco_rl_ur5_b200.parallel import env_seed, shard_range

    for n, w in [(4096, 1), (4096, 8), (10, 4), (7, 8)]:
        r = [shard_range(n, k, w) for k in range(w)]
        assert r[0][0] == 0 and r[-1][1] == n and all(r[i][1] == r[i + 1][0] for i in range(w - 1))
    assert env_seed(shard_range(4096, 3, 8)[0]) == 20000 + 1536


_GLOO_SCRIPT = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["REPO"])
from mujoco_rl_ur5_b200.parallel import shard_range, env_seed, gather_results
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
N = 11
a, b = shard_range(N, rank, world)
idx = torch.arange(a, b)
# a per-env "result" that only depends on the global index (as the engine's results do)
reward = (idx % 2).to(torch.uint8); result = (idx * 3).to(torch.int32); steps = torch.tensor([env_seed(int(i)) for i in idx], dtype=torch.int32)
R, S, T = gather_results(reward, result, steps, N)
g = torch.arange(N)
assert torch.equal(R, (g % 2).to(torch.uint8)) and torch.equal(S, (g * 3).to(torch.int32)) and torch.equal(T, (20000 + g).to(torch.int32))
dist.barrier(); dist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_two_rank_gloo_gather(tmp_path):
    """N>1 host logic on CPU: 2 processes, gloo backend, 127.0.0.1 rendezvous; identical global result on both ranks."""
    script = tmp_path / "gloo_gather.py"
    script.write_text(_GLOO_SCRIPT)
    env = dict(os.environ, REPO=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29533",
           str(script)]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=240)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("ok") == 2


def test_recorded_grasp_issues_the_reference_movement_sequence(tmp_path):
    """record_grasps=True path of the façade (GraspingEnv.py:205-386 issued phase by phase so the side-camera picture can be taken
    between the final finger check and the re-opening, :329-335): call order, targets, step budgets and tolerances against the
    reference function, with a scripted controller (no GPU)."""
    import sys

    sys.path.insert(0, os.path.join(ROOT, "mujoco_rl_ur5_b200", "compat"))
    from mujoco_rl_ur5_b200.grasp_env import GraspEnv

    class Gain:
        Kp = 20.0

    class Fake:
        def __init__(self, script):
            self.calls, self.script = [], script
            self.actuators = [[None, None, None, None, Gain()]]
            self.current_target_joint_values = np.zeros(7)

        def _r(self, name, default="success"):
            return self.script.get(name, default)

        def move_ee(self, xyz, max_steps=None, tolerance=None, **kw):
            self.calls.append(("move_ee", [round(float(v), 4) for v in xyz], max_steps, tolerance))
            return self._r("move_ee%d" % sum(c[0] == "move_ee" for c in self.calls))

        def move_group_to_joint_target(self, tolerance=None, max_steps=None, **kw):
            self.calls.append(("wrist", round(float(self.current_target_joint_values[5]), 4), max_steps, tolerance))
            return "success"

        def open_gripper(self, half=False, **kw):
            self.calls.append(("open", half, self.actuators[0][4].Kp))
            return "success"

        def grasp(self, **kw):
            self.calls.append(("grasp",))
            return self._r("grasp", True)

        def close_gripper(self, max_steps=None, **kw):
            self.calls.append(("close", max_steps))
            return self._r("close", "max. steps reached: 1000")

        def stay(self, ms, **kw):
            self.calls.append(("stay", ms))

        def get_image_data(self, width=200, height=200, camera="top_down", **kw):
            self.calls.append(("image", camera, width, height))
            img = np.zeros((height, width, 3), np.uint8)
            img[..., 0] = 200
            return img, np.zeros((height, width), np.float32)

    def make(script):
        e = GraspEnv.__new__(GraspEnv)
        e.controller, e.rotations, e.TABLE_HEIGHT, e.grasp_counter, e.quiet, e.render = Fake(script), {0: 0, 3: 90}, 0.91, 0, True, False
        return e

    # a successful grasp: picture taken after the 1000-step finger check and before the gripper opens
    e = make({})
    ok, png = e.move_and_grasp_recorded(np.array([0.1, -0.55, 0.95]), 3, directory=str(tmp_path))
    names = [c[0] for c in e.controller.calls]
    assert ok and names == ["move_ee", "wrist", "open", "move_ee", "stay", "grasp", "move_ee", "move_ee", "close", "image", "open", "stay", "wrist"]
    c = e.controller.calls
    assert c[0] == ("move_ee", [0.1, -0.55, 1.1], 1000, 0.05) and c[1] == ("wrist", round(np.pi / 2, 4), 500, 0.05) and c[2][:2] == ("open", True)
    assert c[3] == ("move_ee", [0.1, -0.55, 0.94], 300, 0.01) and c[4] == ("stay", 100)
    assert c[6] == ("move_ee", [0.0, -0.6, 1.1], 1000, 0.05) and c[7] == ("move_ee", [0.6, 0.0, 1.15], 1200, 0.01)
    assert c[8] == ("close", 1000) and c[9] == ("image", "side", 1000, 1000) and c[10] == ("open", False, 10.0) and c[11] == ("stay", 200)
    assert c[12][1] == 0.0 and e.controller.actuators[0][4].Kp == 20.0
    from PIL import Image

    im = Image.open(png)
    assert os.path.basename(png) == "Grasp_1.png" and im.size == (1000, 1000) and im.getpixel((5, 5)) == (200, 0, 0)
    # grasp height clamps at the table; unreachable target falls back to the centre; a stuck approach skips the attempt
    e = make({"move_ee1": "No valid joint angles received, could not move EE to position.", "grasp": False})
    ok, png = e.move_and_grasp_recorded(np.array([0.3, -0.9, 0.90]), 0, directory=str(tmp_path))
    c = e.controller.calls
    assert not ok and png is None and c[1] == ("move_ee", [0.0, -0.6, 1.1], 1000, 0.05) and c[4] == ("move_ee", [0.3, -0.9, 0.91], 300, 0.01)
    assert "close" not in [x[0] for x in c] and "image" not in [x[0] for x in c]
    e = make({"move_ee1": "max. steps reached: 1000"})
    ok, _ = e.move_and_grasp_recorded(np.array([0.0, -0.6, 0.95]), 0, directory=str(tmp_path))
    assert not ok and [x[0] for x in e.controller.calls] == ["move_ee", "move_ee", "move_ee", "open", "wrist"]
    # object lost on the way to the drop position: the finger check closes completely ("success") -> no reward, no picture
    e = make({"close": "success"})
    ok, png = e.move_and_grasp_recorded(np.array([0.0, -0.6, 0.95]), 0, directory=str(tmp_path))
    assert not ok and png is None and ("stay", 200) not in e.controller.calls
