"""TEST INFRASTRUCTURE: ctypes binding of the CPU oracle (oracle/grasp_oracle.c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build():
    subprocess.check_call(["make", "-s", "-C", _DIR])


def lib():
    global _LIB
    if _LIB is None:
        # GRASP_ORACLE_SO: another build of the same source (e.g. -ffp-contract=fast) for rounding-sensitivity experiments
        so = os.environ.get("GRASP_ORACLE_SO")
        if not so:
            so = os.path.join(_DIR, "libgrasp_oracle.so")
            if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(os.path.join(_DIR, "grasp_oracle.c")):
                build()
        L = C.CDLL(so)
        P, D, I = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_model_load.restype = P
        L.orc_model_load.argtypes = [C.c_char_p, C.c_int64]
        L.orc_model_free.argtypes = [P]
        L.orc_model_size.argtypes = [P, C.c_int]
        L.orc_env_create.restype = P
        L.orc_env_create.argtypes = [P]
        L.orc_env_free.argtypes = [P]
        for f in ("orc_forward", "orc_step", "orc_fk"):
            getattr(L, f).argtypes = [P]
        for f in ("orc_qpos", "orc_qvel", "orc_qacc_ws", "orc_ctrl", "orc_target", "orc_kp", "orc_last_input"):
            getattr(L, f).restype = D
            getattr(L, f).argtypes = [P]
        L.orc_substeps.restype = C.c_long
        L.orc_substeps.argtypes = [P]
        L.orc_set_dt_pid.argtypes = [P, C.c_double]
        L.orc_set_solver.argtypes = [P, C.c_int]
        L.orc_set_maxcon.argtypes = [P, C.c_int]
        L.orc_con_overflow.argtypes = [P]
        L.orc_set_maxsr.argtypes = [P, C.c_int]
        L.orc_sr_overflow.argtypes = [P]
        L.orc_efc_split.argtypes = [P, I]
        L.orc_ncand.argtypes = [P]
        L.orc_ncon_peak.argtypes = [P, C.c_int]
        L.orc_reset.argtypes = [P, D, D]
        L.orc_field.restype = D
        L.orc_field.argtypes = [P, C.c_char_p, I]
        for f in ("orc_ncon", "orc_nefc", "orc_solver_iter"):
            getattr(L, f).argtypes = [P]
        L.orc_contact.argtypes = [P, C.c_int, D]
        L.orc_move_group.argtypes = [P, C.c_int, D, C.c_int, C.c_double, C.c_int, I]
        L.orc_stay.argtypes = [P, C.c_int]
        L.orc_ik.argtypes = [P, D, D]
        L.orc_move_ee.argtypes = [P, D, C.c_double, C.c_int, I]
        L.orc_move_and_grasp.argtypes = [P, D, C.c_int, C.c_double, I]
        L.orc_pixel_2_world.argtypes = [P, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, D]
        L.orc_depth_2_meters.restype = C.c_double
        L.orc_depth_2_meters.argtypes = [P, C.c_double]
        L.orc_render.argtypes = [P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_float)]
        L.orc_render_probe.argtypes = [P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64), C.c_double, C.c_double, I, I]
        L.orc_newton_stats.argtypes = [C.POINTER(C.c_long), C.c_int]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def newton_stats(reset=True):
    """process-wide solver statistics of the oracle (profiling aid): dict with solves, Hessian builds, builds whose active set did not
    change since the previous build of the same solve, line-search iterations, constraint rows, solves ending after 1 / 2 / 3+ builds"""
    out = (C.c_long * 8)()
    lib().orc_newton_stats(out, 1 if reset else 0)
    keys = ["solves", "builds", "builds_same_active_set", "linesearch_iterations", "rows", "solves_1_build", "solves_2_builds", "solves_3plus_builds"]
    return dict(zip(keys, [int(v) for v in out]))


class OracleEnv:
    """One fp64 CPU environment."""

    GROUPS = {"All": 0x7F, "Arm": 0x1F, "Gripper": 0x40}

    def __init__(self, blob: bytes):
        L = lib()
        self.L = L
        self.model = L.orc_model_load(blob, len(blob))
        assert self.model, "oracle could not load the model blob"
        self.env = L.orc_env_create(self.model)
        self.nq, self.nv, self.nbody, self.ngeom, self.nM, self.njnt = [L.orc_model_size(self.model, k) for k in range(6)]

    def close(self):
        if self.env:
            self.L.orc_env_free(self.env)
            self.L.orc_model_free(self.model)
            self.env = None

    def _view(self, fn, n):
        return np.ctypeslib.as_array(getattr(self.L, fn)(self.env), shape=(n,))

    @property
    def qpos(self):
        return self._view("orc_qpos", self.nq)

    @property
    def qvel(self):
        return self._view("orc_qvel", self.nv)

    @property
    def qacc_warmstart(self):
        return self._view("orc_qacc_ws", self.nv)

    @property
    def ctrl(self):
        return self._view("orc_ctrl", 7)

    @property
    def target(self):
        return self._view("orc_target", 7)

    @property
    def kp(self):
        return self._view("orc_kp", 7)

    @property
    def last_input(self):
        return self._view("orc_last_input", 7)

    @property
    def substeps(self):
        return int(self.L.orc_substeps(self.env))

    def reset(self, qpos, qvel=None):
        qpos = np.ascontiguousarray(qpos, np.float64)
        qv = None if qvel is None else _dp(np.ascontiguousarray(qvel, np.float64))
        self.L.orc_reset(self.env, _dp(qpos), qv)

    def set_solver(self, name):
        self.L.orc_set_solver(self.env, {"newton": 0, "pgs": 1}[name])

    def set_maxcon(self, n):
        """contact capacity (default 256): later contacts of the emission order (analytic pairs, then MPR pairs, both in pair
        order) are dropped and `con_overflow` is set, as in the CUDA engine's list of GE_MAXCON contacts"""
        self.L.orc_set_maxcon(self.env, int(n))

    @property
    def con_overflow(self):
        """1 if the last collision stage found more contacts than the capacity"""
        return int(self.L.orc_con_overflow(self.env))

    def set_maxsr(self, n=-1):
        """simple-row capacity: the equality rows and then the first limit rows (joint order, lower side first) up to n rows in all
        are kept, later limit rows are dropped and `sr_overflow` is set, as in the CUDA engine's GE_MAXSR slots (n < 0: no cap)"""
        self.L.orc_set_maxsr(self.env, int(n))

    @property
    def sr_overflow(self):
        """1 if the last forward() dropped limit rows at the simple-row capacity"""
        return int(self.L.orc_sr_overflow(self.env))

    @property
    def efc_split(self):
        """constraint rows of the last forward(): (equality, joint limit, contact)"""
        out = (C.c_int * 3)()
        self.L.orc_efc_split(self.env, out)
        return tuple(int(v) for v in out)

    @property
    def ncand(self):
        """pairs that passed the broad phase in the last collision stage"""
        return int(self.L.orc_ncand(self.env))

    def ncon_peak(self, reset=True):
        """the most contacts one collision stage found since the previous call with reset=True, counting those beyond the capacity"""
        return int(self.L.orc_ncon_peak(self.env, 1 if reset else 0))

    def boxbox(self):
        """one row per box-box pair the last collision stage tested (col_box_box): geom1, geom2, outcome (0 separated, 1 face contact,
        2 edge-edge), reference box (1 or 2, 0 unless a face contact), best face axis (0-2 box 1, 3-5 box 2), face axes whose
        separation ties the best bit for bit, edge axes skipped by the 1e-6 guard with a non-zero cross product, incident vertices
        exactly on a clip line, contacts emitted; int array [n, 9]"""
        return self.field("boxbox").reshape(-1, 9).astype(np.int64)

    def forward(self):
        self.L.orc_forward(self.env)

    def step(self, n=1):
        for _ in range(n):
            self.L.orc_step(self.env)

    def fk(self):
        self.L.orc_fk(self.env)

    def field(self, name):
        n = C.c_int(0)
        p = self.L.orc_field(self.env, name.encode(), C.byref(n))
        if not p or n.value == 0:
            return np.zeros(0)
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    @property
    def ncon(self):
        return self.L.orc_ncon(self.env)

    @property
    def nefc(self):
        return self.L.orc_nefc(self.env)

    @property
    def solver_iter(self):
        return self.L.orc_solver_iter(self.env)

    def contacts(self):
        out = np.zeros((self.ncon, 16))
        for i in range(self.ncon):
            self.L.orc_contact(self.env, i, _dp(out[i]))
        return out

    def dense_M(self, dof_parentid, dof_Madr, which="qM"):
        q = self.field(which)
        nv = self.nv
        M = np.zeros((nv, nv))
        for i in range(nv):
            j, k = i, 0
            while j >= 0:
                M[i, j] = M[j, i] = q[dof_Madr[i] + k]
                j = dof_parentid[j]
                k += 1
        return M

    def move_group(self, group="All", target=None, tolerance=0.1, max_steps=10000):
        mask = self.GROUPS[group] if isinstance(group, str) else int(group)
        steps = C.c_int(0)
        if target is None:
            r = self.L.orc_move_group(self.env, mask, None, 0, tolerance, max_steps, C.byref(steps))
        else:
            t = np.ascontiguousarray(target, np.float64)
            r = self.L.orc_move_group(self.env, mask, _dp(t), 1, tolerance, max_steps, C.byref(steps))
        return r, steps.value

    def stay(self, ms):
        self.L.orc_stay(self.env, int(ms))

    def ik(self, xyz):
        q5 = np.zeros(5)
        ok = self.L.orc_ik(self.env, _dp(np.ascontiguousarray(xyz, np.float64)), _dp(q5))
        return (q5 if ok else None)

    def move_ee(self, xyz, tolerance=0.05, max_steps=1000):
        steps = C.c_int(0)
        r = self.L.orc_move_ee(self.env, _dp(np.ascontiguousarray(xyz, np.float64)), tolerance, max_steps, C.byref(steps))
        return r, steps.value

    def move_and_grasp(self, coords, rot, table_height=0.91):
        info = (C.c_int * 12)()
        r = self.L.orc_move_and_grasp(self.env, _dp(np.ascontiguousarray(coords, np.float64)), int(rot), table_height, info)
        return int(r), list(info)

    def pixel_2_world(self, px, py, depth, cam=1, W=200, H=200):
        out = np.zeros(3)
        self.L.orc_pixel_2_world(self.model, cam, W, H, float(px), float(py), float(depth), _dp(out))
        return out

    def depth_2_meters(self, gl_depth):
        return float(self.L.orc_depth_2_meters(self.model, float(gl_depth)))

    def render(self, cam=1, W=200, H=200):
        rgb = np.zeros((H, W, 3), np.uint8)
        depth = np.zeros((H, W), np.float32)
        self.L.orc_render(self.env, cam, W, H, rgb.ctypes.data_as(C.POINTER(C.c_uint8)), depth.ctypes.data_as(C.POINTER(C.c_float)))
        return rgb, depth

    # flag bits of render_probe
    PROBE_MOVES, PROBE_TIE, PROBE_RGB_ROUNDING, PROBE_F32_ROUNDING, PROBE_CHECKER = 1, 2, 4, 8, 16

    def render_probe(self, cam, W, H, pixels=None, eps_px=1e-10, eps_m=1e-13):
        """where rounding may decide a pixel of render(cam, W, H): for the flat pixel indices r * W + c (None: all), the geom render()
        shows there (-1: background) and a bit set of reasons a renderer computing the same fp64 expressions with other rounding may
        show something else (orc_render_probe in grasp_oracle.c).  Returns (gid, flags), int32 arrays shaped like `pixels`."""
        pix = np.arange(W * H, dtype=np.int64) if pixels is None else np.ascontiguousarray(pixels, np.int64).ravel()
        gid = np.zeros(len(pix), np.int32)
        flags = np.zeros(len(pix), np.int32)
        I = C.POINTER(C.c_int)
        self.L.orc_render_probe(self.env, cam, W, H, len(pix), pix.ctypes.data_as(C.POINTER(C.c_int64)), float(eps_px), float(eps_m),
                                gid.ctypes.data_as(I), flags.ctypes.data_as(I))
        shape = (H, W) if pixels is None else np.shape(pixels)
        return gid.reshape(shape), flags.reshape(shape)
