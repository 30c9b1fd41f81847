"""Shared helpers for the parity tests: deterministic resets and action replays (SURVEY 8(d) seeds)."""
import numpy as np

HOME = np.array([0, -1.57, 1.57, -1.57, -1.57, 0.0, 0.3])  # GraspingEnv.py:418


def reset_qpos_scene_a(A, env_index):
    """Scene-A reset = the commented IT4 rule (GraspingEnv.py:435-463): x~U(-.25,.25), y~U(-.17,.17), z=0, identity quat;
    RNG = RandomState(20000 + env_index), objects in joint order, draws x then y."""
    rng = np.random.RandomState(20000 + env_index)
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3  # right knuckle follows the equality constraint
    nobj = (int(np.asarray(A["nq"]).ravel()[0]) - 8) // 7
    for i in range(nobj):
        a = 8 + 7 * i
        q[a] = rng.uniform(-0.25, 0.25)
        q[a + 1] = rng.uniform(-0.17, 0.17)
        q[a + 2] = 0.0
        q[a + 3:a + 7] = [1, 0, 0, 0]
    return q


def object_positions(A, qpos):
    nobj = (int(np.asarray(A["nq"]).ravel()[0]) - 8) // 7
    first = int(np.asarray(A["nbody"]).ravel()[0]) - nobj
    return np.array([qpos[8 + 7 * i:11 + 7 * i] + A["body_pos"][first + i] for i in range(nobj)])


def contact_is_analytic(A, contacts):
    """per contact row (geom ids in columns 13, 14): True if its pair has a closed-form narrow phase, False if it goes through MPR
    (the oracle's and the engine's pair_is_analytic; geom types 0 plane, 2 sphere, 3 capsule, 5 cylinder, 6 box, 7 mesh)"""
    gtype = np.asarray(A["geom_type"]).ravel()
    out = []
    for g1, g2 in np.asarray(contacts)[:, 13:15].astype(int):
        t1, t2 = int(gtype[g1]), int(gtype[g2])
        out.append(t1 == 0 or (t1 == 2 and t2 in (2, 3, 5, 6)) or (t1, t2) in ((6, 6), (3, 3)))
    return np.array(out, bool)


def reset_qpos_scene_b(A, env_index):
    """Scene-B reset = the live rule of GraspingEnv.py:418-430 (x, y, z, then Quaternion.random()'s three uniforms per object),
    RNG = RandomState(20000 + env_index)."""
    rng = np.random.RandomState(20000 + env_index)
    q = np.array(A["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = 0.3
    for i in range(40):
        a = 8 + 7 * i
        q[a] = rng.uniform(-0.25, 0.25)
        q[a + 1] = rng.uniform(-0.77, -0.43)
        q[a + 2] = rng.uniform(1.0, 1.5)
        r1, r2, r3 = rng.random_sample(3)
        q[a + 3:a + 7] = [np.sqrt(1 - r1) * np.sin(2 * np.pi * r2), np.sqrt(1 - r1) * np.cos(2 * np.pi * r2),
                          np.sqrt(r1) * np.sin(2 * np.pi * r3), np.sqrt(r1) * np.cos(2 * np.pi * r3)]
    return q
