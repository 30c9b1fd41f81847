#!/usr/bin/env python
"""Small workload for compute-sanitizer (tools/sanitize.sh): every kernel of libgrasp_engine.so on a handful of environments —
set_state, a movement with contacts (k_run: warp-per-env build for the 6-object scene, CTA-per-env build for the 40-object
scene), open-loop steps, IK, pixel_2_world, body_xpos, render.  Sizes are tiny because racecheck slows kernels down ~100x."""
import sys, os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_rl_ur5_b200.engine import BatchedEngine
from mujoco_rl_ur5_b200.batched_env import scene_a_reset_qpos, scene_b_reset_qpos, HOME
from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

steps_a, steps_b = int(sys.argv[1]) if len(sys.argv) > 1 else 12, int(sys.argv[2]) if len(sys.argv) > 2 else 3
A, _ = load_scene("A")
eng = BatchedEngine(load_scene_blob("A"), 5, 0)   # 5 envs: one full CTA of 4 warps + a partial one
eng.set_state(np.stack([scene_a_reset_qpos(A, 20000 + i) for i in range(5)]))
eng.move_group("All", np.tile(HOME + 0.1, (5, 1)), 1e-7, steps_a)
eng.run()
eng.grasp(np.tile([0.0, -0.6, 0.93], (5, 1)), np.arange(5, dtype=np.int32), 0.91)
eng.run(steps_a)
eng.set_ctrl(np.zeros((5, 7)))
eng.step_open_loop(2)
eng.ik(np.tile([0.0, -0.6, 1.1], (5, 1)))
eng.body_xpos()
rgb, depth = eng.render(1, 64, 64)
print("scene A ok, status", eng.status().cpu().numpy(), "depth range", float(depth.min()), float(depth.max()))
eng.close()
if steps_b > 0:
    B, _ = load_scene("B")
    eng = BatchedEngine(load_scene_blob("B"), 2, 0)
    eng.set_state(np.stack([scene_b_reset_qpos(B, 20000 + i) for i in range(2)]))
    eng.move_group("All", np.tile(HOME, (2, 1)), 1e-7, steps_b)
    eng.run()
    print("scene B ok, status", eng.status().cpu().numpy())
    eng.close()
