"""ctypes binding of libgrasp_engine.so (include/grasp_engine.h) with torch tensors as device buffers.

PyTorch is plumbing here (device memory, streams, torch.distributed); every computation on the hot path is a kernel
of the in-tree CUDA library.  There is NO CPU fallback: if the library is missing or no GPU is visible, constructing a
`BatchedEngine` raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libgrasp_engine.so")
_LIB = None

SYMBOLS = [
    "ge_last_error", "ge_version", "ge_create", "ge_destroy", "ge_size", "ge_set_state", "ge_get_state", "ge_get_body_xpos",
    "ge_set_gain", "ge_set_targets", "ge_get_targets", "ge_move_group", "ge_move_ee", "ge_stay", "ge_grasp", "ge_run", "ge_run_async", "ge_get_results",
    "ge_get_grasp_info", "ge_get_status", "ge_get_busy", "ge_set_ctrl", "ge_get_ctrl", "ge_step_open_loop", "ge_ik", "ge_pixel_2_world", "ge_render", "ge_debug_forward", "ge_counters",
    "ge_snapshot", "ge_restore", "ge_clone",
]
GROUPS = {"All": 0x7F, "Arm": 0x1F, "Gripper": 0x40}
MOVE_RESULT = {0: "", 1: "success", 2: "max. steps reached: {}", 3: "No valid joint angles received, could not move EE to position."}


class EngineError(RuntimeError):
    pass


def load_library():
    """Load the CUDA engine; raises EngineError (never falls back) if it has not been built."""
    global _LIB
    if _LIB is None:
        path = os.environ.get("GE_LIB", LIB_PATH)  # GE_LIB: alternative build of the same library (the -fmad=false test build, profile builds)
        if not os.path.exists(path):
            raise EngineError(f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(path)
        P = C.c_void_p
        L.ge_last_error.restype = C.c_char_p
        L.ge_version.restype = C.c_char_p
        L.ge_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, P, C.POINTER(P)]
        L.ge_destroy.argtypes = [P]
        L.ge_size.argtypes = [P, C.c_int]
        L.ge_set_state.argtypes = [P, P, P, P]
        L.ge_get_state.argtypes = [P, P, P]
        L.ge_get_body_xpos.argtypes = [P, P]
        L.ge_set_gain.argtypes = [P, C.c_int, P, C.c_double]
        L.ge_set_targets.argtypes = [P, P]
        L.ge_get_targets.argtypes = [P, P]
        L.ge_move_group.argtypes = [P, C.c_int, P, C.c_double, C.c_int, P]
        L.ge_move_ee.argtypes = [P, P, C.c_double, C.c_int, P]
        L.ge_stay.argtypes = [P, C.c_int, P]
        L.ge_grasp.argtypes = [P, P, P, C.c_double, P]
        L.ge_run.argtypes = [P, C.c_int, C.POINTER(C.c_int)]
        L.ge_run_async.argtypes = [P, C.c_int]
        L.ge_get_results.argtypes = [P, P, P, P, P]
        L.ge_get_grasp_info.argtypes = [P, P]
        L.ge_get_status.argtypes = [P, P]
        L.ge_get_busy.argtypes = [P, P]
        L.ge_set_ctrl.argtypes = [P, P, P]
        L.ge_get_ctrl.argtypes = [P, P]
        L.ge_step_open_loop.argtypes = [P, C.c_int, P]
        L.ge_ik.argtypes = [P, P, P, P]
        L.ge_pixel_2_world.argtypes = [P, C.c_int, C.c_int, C.c_int, P, P, P, P]
        L.ge_render.argtypes = [P, C.c_int, C.c_int, C.c_int, P, P]
        L.ge_debug_forward.argtypes = [P, C.c_int, C.c_char_p, C.POINTER(C.c_double), C.c_int]
        L.ge_counters.argtypes = [P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.ge_snapshot.argtypes = [P, P, C.c_int, P]
        L.ge_restore.argtypes = [P, P, C.c_int, P]
        L.ge_clone.argtypes = [P, P]
        _LIB = L
    return _LIB


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class BatchedEngine:
    """N independent copies of one compiled scene on one GPU (structure-of-arrays state in HBM)."""

    def __init__(self, blob: bytes, n_envs: int, device: int = 0):
        import torch

        if not torch.cuda.is_available():
            raise EngineError("BatchedEngine needs a CUDA device (there is no CPU fallback)")
        self.torch = torch
        self.L = load_library()
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.current_stream(self.device)
        h = C.c_void_p()
        r = self.L.ge_create(blob, len(blob), int(n_envs), device, C.c_void_p(self.stream.cuda_stream), C.byref(h))
        if r != 0:
            raise EngineError(f"ge_create failed ({r}): {self.L.ge_last_error().decode()}")
        self.h = h
        self.n_envs = int(n_envs)
        self.nq, self.nv, self.nbody, self.ngeom, self.nu = [self.L.ge_size(h, k) for k in range(5)]
        self.smem_bytes = self.L.ge_size(h, 7)
        self._blob, self._fingerprint = blob, None

    def size(self, what):
        """ge_size: 0 nq, 1 nv, 2 nbody, 3 ngeom, 4 nu, 5 n_envs, 6 max contacts, 7 workspace bytes per env, 8 envs per CTA,
        9 workspace placement (0 shared memory, 1 HBM rows), 10 doubles of the Newton Hessian block region in the workspace (hcap),
        11 doubles of a full packed Hessian = of one env's HBM overflow row (hfull), 12 envs of the sub-step kernel resident per SM
        (occupancy API), 13 Newton Hessian builds that used the overflow row since creation"""
        return int(self.L.ge_size(self.h, int(what)))

    # ------------------------------------------------------------------ helpers
    def _ck(self, r, what):
        if r < 0:
            raise EngineError(f"{what} failed ({r}): {self.L.ge_last_error().decode()}")
        return r

    def _dev(self, a, dtype):
        t = self.torch
        if a is None:
            return None
        if not isinstance(a, t.Tensor):
            a = t.as_tensor(np.ascontiguousarray(a))
        return a.to(device=self.device, dtype=dtype, non_blocking=True).contiguous()

    def close(self):
        if getattr(self, "h", None):
            self.L.ge_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ state
    def set_state(self, qpos, qvel=None, env_mask=None):
        t = self.torch
        qpos = self._dev(qpos, t.float64).reshape(self.n_envs, self.nq)
        qvel = None if qvel is None else self._dev(qvel, t.float64).reshape(self.n_envs, self.nv)
        env_mask = self._dev(env_mask, t.uint8)
        self._ck(self.L.ge_set_state(self.h, _ptr(qpos), _ptr(qvel), _ptr(env_mask)), "ge_set_state")
        self._keep = (qpos, qvel, env_mask)

    def get_state(self):
        t = self.torch
        qpos = t.empty((self.n_envs, self.nq), dtype=t.float64, device=self.device)
        qvel = t.empty((self.n_envs, self.nv), dtype=t.float64, device=self.device)
        self._ck(self.L.ge_get_state(self.h, _ptr(qpos), _ptr(qvel)), "ge_get_state")
        return qpos, qvel

    # ------------------------------------------------------------------ whole environment states (env_state.py, format "GES1")
    @property
    def state_bytes(self):
        """bytes of one environment state record (ge_size 14)"""
        return self.size(14)

    @property
    def fingerprint(self):
        """FNV-1a-64 of the model blob, as the engine writes it into every record"""
        if self._fingerprint is None:
            from .env_state import fingerprint

            self._fingerprint = fingerprint(self._blob)
        return self._fingerprint

    def snapshot(self, envs=None):
        """EngineState with one record per env of `envs` (indices, default all), on this engine's device"""
        from .env_state import EngineState

        t = self.torch
        ids = None if envs is None else self._dev(envs, t.int32).reshape(-1)
        n = self.n_envs if ids is None else ids.numel()
        rec = t.empty((n, self.state_bytes), dtype=t.uint8, device=self.device)
        self._ck(self.L.ge_snapshot(self.h, _ptr(ids), n, _ptr(rec)), "ge_snapshot")
        self._keep = ids
        return EngineState(rec, self.nq, self.nv, self.fingerprint)

    def restore(self, state, rows=None):
        """env e <- record rows[e] of `state` (-1: leave env e alone; default: record e).  Raises EngineError, with the engine left
        unchanged, for a record of another scene (GE_ERR_STATE) or a row outside [-1, len(state))"""
        t = self.torch
        if state.record_bytes != self.state_bytes:  # the library reads [n, R] records with its own R: refuse before it reads
            raise EngineError(f"ge_restore refused: records of {state.record_bytes} bytes, this scene's are {self.state_bytes}")
        rec = state.data.to(self.device).contiguous()
        rows = None if rows is None else self._dev(rows, t.int32).reshape(self.n_envs)
        self._ck(self.L.ge_restore(self.h, _ptr(rec), len(state), _ptr(rows)), "ge_restore")
        self._keep = (rec, rows)

    def clone(self, src):
        """env e <- the state env src[e] had before the call (-1: keep); src [N]"""
        src = self._dev(src, self.torch.int32).reshape(self.n_envs)
        self._ck(self.L.ge_clone(self.h, _ptr(src)), "ge_clone")
        self._keep = src

    def body_xpos(self):
        t = self.torch
        x = t.empty((self.n_envs, self.nbody, 3), dtype=t.float64, device=self.device)
        self._ck(self.L.ge_get_body_xpos(self.h, _ptr(x)), "ge_get_body_xpos")
        return x

    def set_gain(self, actuator, value):
        t = self.torch
        if np.isscalar(value):
            self._ck(self.L.ge_set_gain(self.h, actuator, None, float(value)), "ge_set_gain")
        else:
            kp = self._dev(value, t.float64)
            self._ck(self.L.ge_set_gain(self.h, actuator, _ptr(kp), 0.0), "ge_set_gain")
            self._keep = kp

    def set_targets(self, target):
        t = self.torch
        tg = self._dev(target, t.float64).reshape(self.n_envs, 7)
        self._ck(self.L.ge_set_targets(self.h, _ptr(tg)), "ge_set_targets")
        self._keep = tg

    def get_targets(self):
        t = self.torch
        tg = t.empty((self.n_envs, 7), dtype=t.float64, device=self.device)
        self._ck(self.L.ge_get_targets(self.h, _ptr(tg)), "ge_get_targets")
        return tg

    # ------------------------------------------------------------------ movements
    def move_group(self, group="All", target=None, tolerance=0.1, max_steps=10000, env_mask=None):
        t = self.torch
        mask = GROUPS[group] if isinstance(group, str) else int(group)
        full = None
        if target is not None:
            tg = self._dev(target, t.float64).reshape(self.n_envs, -1)
            ids = [i for i in range(7) if mask >> i & 1]
            if tg.shape[1] == 7:
                full = tg
            else:
                assert tg.shape[1] == len(ids), "Mismatching target dimensions for group"
                full = t.zeros((self.n_envs, 7), dtype=t.float64, device=self.device)
                full[:, ids] = tg
        env_mask = self._dev(env_mask, t.uint8)
        self._ck(self.L.ge_move_group(self.h, mask, _ptr(full), float(tolerance), int(max_steps), _ptr(env_mask)), "ge_move_group")
        self._keep = (full, env_mask)

    def move_ee(self, xyz, tolerance=0.05, max_steps=1000, env_mask=None):
        t = self.torch
        xyz = self._dev(xyz, t.float64).reshape(self.n_envs, 3)
        env_mask = self._dev(env_mask, t.uint8)
        self._ck(self.L.ge_move_ee(self.h, _ptr(xyz), float(tolerance), int(max_steps), _ptr(env_mask)), "ge_move_ee")
        self._keep = (xyz, env_mask)

    def stay(self, ms, env_mask=None):
        env_mask = self._dev(env_mask, self.torch.uint8)
        self._ck(self.L.ge_stay(self.h, int(ms), _ptr(env_mask)), "ge_stay")
        self._keep = env_mask

    def grasp(self, coords, rot, table_height=0.91, env_mask=None):
        t = self.torch
        coords = self._dev(coords, t.float64).reshape(self.n_envs, 3)
        rot = self._dev(rot, t.int32).reshape(self.n_envs)
        env_mask = self._dev(env_mask, t.uint8)
        self._ck(self.L.ge_grasp(self.h, _ptr(coords), _ptr(rot), float(table_height), _ptr(env_mask)), "ge_grasp")
        self._keep = (coords, rot, env_mask)

    def run(self, max_substeps=0):
        busy = C.c_int(0)
        self._ck(self.L.ge_run(self.h, int(max_substeps), C.byref(busy)), "ge_run")
        return busy.value

    def run_async(self, substeps):
        self._ck(self.L.ge_run_async(self.h, int(substeps)), "ge_run_async")

    def results(self):
        t = self.torch
        N = self.n_envs
        result = t.empty(N, dtype=t.int32, device=self.device)
        steps = t.empty(N, dtype=t.int32, device=self.device)
        reward = t.empty(N, dtype=t.uint8, device=self.device)
        total = t.empty(N, dtype=t.int64, device=self.device)
        self._ck(self.L.ge_get_results(self.h, _ptr(result), _ptr(steps), _ptr(reward), _ptr(total)), "ge_get_results")
        return result, steps, reward, total

    def grasp_info(self):
        t = self.torch
        info = t.empty((self.n_envs, 12), dtype=t.int32, device=self.device)
        self._ck(self.L.ge_get_grasp_info(self.h, _ptr(info)), "ge_get_grasp_info")
        return info

    def status(self):
        t = self.torch
        st = t.empty(self.n_envs, dtype=t.int32, device=self.device)
        self._ck(self.L.ge_get_status(self.h, _ptr(st)), "ge_get_status")
        return st

    def busy(self):
        t = self.torch
        b = t.empty(self.n_envs, dtype=t.uint8, device=self.device)
        self._ck(self.L.ge_get_busy(self.h, _ptr(b)), "ge_get_busy")
        return b

    def set_ctrl(self, ctrl, env_mask=None):
        """sim.data.ctrl[:] = ctrl for all 7 actuators ([N,7]); the values stay until the next PID evaluation overwrites them"""
        t = self.torch
        c = self._dev(ctrl, t.float64).reshape(self.n_envs, 7)
        env_mask = self._dev(env_mask, t.uint8)
        self._ck(self.L.ge_set_ctrl(self.h, _ptr(c), _ptr(env_mask)), "ge_set_ctrl")
        self._keep = (c, env_mask)

    def get_ctrl(self):
        t = self.torch
        c = t.empty((self.n_envs, 7), dtype=t.float64, device=self.device)
        self._ck(self.L.ge_get_ctrl(self.h, _ptr(c)), "ge_get_ctrl")
        return c

    def step_open_loop(self, substeps=1, env_mask=None):
        """`substeps` bare sim.step() calls with the current controls (no PID)"""
        env_mask = self._dev(env_mask, self.torch.uint8)
        self._ck(self.L.ge_step_open_loop(self.h, int(substeps), _ptr(env_mask)), "ge_step_open_loop")
        self._keep = env_mask

    # ------------------------------------------------------------------ camera / IK
    def ik(self, xyz):
        t = self.torch
        xyz = self._dev(xyz, t.float64).reshape(self.n_envs, 3)
        q5 = t.empty((self.n_envs, 5), dtype=t.float64, device=self.device)
        ok = t.empty(self.n_envs, dtype=t.uint8, device=self.device)
        self._ck(self.L.ge_ik(self.h, _ptr(xyz), _ptr(q5), _ptr(ok)), "ge_ik")
        return q5, ok

    def pixel_2_world(self, px, py, depth, cam=1, width=200, height=200):
        t = self.torch
        px = self._dev(px, t.int32)
        py = self._dev(py, t.int32)
        depth = self._dev(depth, t.float32)
        xyz = t.empty((self.n_envs, 3), dtype=t.float64, device=self.device)
        self._ck(self.L.ge_pixel_2_world(self.h, cam, width, height, _ptr(px), _ptr(py), _ptr(depth), _ptr(xyz)), "ge_pixel_2_world")
        return xyz

    def render(self, cam=1, width=200, height=200, out=None):
        t = self.torch
        if out is None:
            rgb = t.empty((self.n_envs, height, width, 3), dtype=t.uint8, device=self.device)
            depth = t.empty((self.n_envs, height, width), dtype=t.float32, device=self.device)
        else:
            rgb, depth = out
        self._ck(self.L.ge_render(self.h, cam, width, height, _ptr(rgb), _ptr(depth)), "ge_render")
        return rgb, depth

    # ------------------------------------------------------------------ diagnostics
    def debug_forward(self, env, field, cap=1 << 16):
        """ge_debug_forward: one forward pass of env `env` on its current state, one internal field copied out (names and layouts in
        include/grasp_engine.h; "status", "ncand", "nmpr" and "hlayout" describe the contact list and the last Newton Hessian build)"""
        buf = (C.c_double * cap)()
        n = self._ck(self.L.ge_debug_forward(self.h, int(env), field.encode(), buf, cap), "ge_debug_forward")
        return np.array(buf[:n], dtype=np.float64)

    def counters(self):
        a, b = C.c_int64(0), C.c_int64(0)
        self.L.ge_counters(self.h, C.byref(a), C.byref(b))
        return a.value, b.value
