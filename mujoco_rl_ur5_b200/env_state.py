"""Environment state records of the batched engine: format "GES1" (include/grasp_engine.h, ge_snapshot / ge_restore / ge_clone).

One record of R bytes per environment holds everything that decides how the environment continues: qpos, qvel, the Newton warm start,
the PID block, the pending movement command and grasp-program state, reward, status and the sub-step counter.  `EngineState` keeps
[n, R] records as a u8 tensor (on the device after `BatchedEngine.snapshot`), gives typed views of each field, packs records on the host
from plain field values (handing a state over from the fp64 oracle), and saves / loads them.
"""
import numpy as np

MAGIC = 0x31534547  # "GES1"
INT_FIELDS = ("cmd_active", "cmd_mask", "cmd_maxsteps", "cmd_steps", "cmd_result", "prog_phase", "prog_rot", "prog_grasp", "prog_aux",
              "prog_info", "status", "reward")
# per-env rows of the engine (EnvArrays, csrc/ge_model.cuh) that a record leaves out, and why
EXCLUDED = {
    "busy_count": "ge_run's count of busy envs: set and read within one ge_run",
    "lock": "sub-step kernel scheduling: 0 between launches",
    "owed": "sub-step kernel scheduling: 0 between launches",
    "done": "sub-step kernel scheduling: reset at the start of every launch",
    "ticket": "sub-step kernel scheduling: orders the tasks of one launch relative to a base the host keeps",
    "gws": "Hessian overflow rows: scratch of one Newton Hessian build, written before they are read",
}
# the ctl row: PID target[8] last_input[8] kp[8] ctrl[8] (7 actuators used)
CTL_TARGET, CTL_LAST, CTL_KP, CTL_CTRL = 0, 8, 16, 24


def record_layout(nq, nv):
    """field name -> (numpy dtype, byte offset, shape) of one record; mirrors include/grasp_engine.h"""
    out = {"magic": (np.uint32, 0, ()), "size": (np.uint32, 4, ()), "fingerprint": (np.uint64, 8, ())}
    o = 16
    for name, n in (("qpos", nq), ("qvel", nv), ("qaccws", nv), ("ctl", 32), ("cmd_tol", 0), ("prog_coords", 3), ("prog_table", 0)):
        out[name] = (np.float64, o, (n,) if n else ())
        o += 8 * max(n, 1)
    out["substeps"] = (np.int64, o, ())
    o += 8
    for name in INT_FIELDS:
        n = 12 if name == "prog_info" else 0
        out[name] = (np.int32, o, (n,) if n else ())
        o += 4 * max(n, 1)
    return out


def record_size(nq, nv):
    """R: bytes of one record, padded to a multiple of 128 (= ge_size(h, 14))"""
    dt, off, shape = record_layout(nq, nv)["reward"]
    return (off + 4 + 127) // 128 * 128


def fingerprint(blob):
    """FNV-1a-64 of the model blob's bytes: the model identity every record carries"""
    h = 0xCBF29CE484222325
    for b in bytes(blob):
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


class EngineState:
    """[n, R] state records (u8 tensor `data`) of a scene with `nq` / `nv`, for the model with `fingerprint`.  `facade`: what a
    BatchedGraspEnv keeps beside the engine (observation, step counter, episode), or None for a bare engine snapshot."""

    def __init__(self, data, nq, nv, fingerprint, facade=None):
        import torch

        if data.dtype != torch.uint8 or data.dim() != 2 or data.shape[1] != record_size(nq, nv):
            raise ValueError(f"state records must be u8 [n, {record_size(nq, nv)}], got {tuple(data.shape)} {data.dtype}")
        self.data, self.nq, self.nv, self.fingerprint, self.facade = data, int(nq), int(nv), int(fingerprint), facade

    def __len__(self):
        return self.data.shape[0]

    @property
    def record_bytes(self):
        return self.data.shape[1]

    def field(self, name):
        """view [n, *shape] of one field of every record (writes go to the records)"""
        import torch

        dt, off, shape = record_layout(self.nq, self.nv)[name]
        tdt = {np.uint32: torch.int32, np.uint64: torch.int64, np.float64: torch.float64, np.int64: torch.int64, np.int32: torch.int32}[dt]
        size = int(np.prod(shape, dtype=np.int64)) * np.dtype(dt).itemsize
        return self.data[:, off:off + size].view(tdt).reshape((len(self),) + shape)

    def fields(self, i):
        """record i as a dict of numpy values (host), header included"""
        raw = self.data[i].cpu().numpy()
        out = {}
        for name, (dt, off, shape) in record_layout(self.nq, self.nv).items():
            n = int(np.prod(shape, dtype=np.int64))
            v = raw[off:off + n * np.dtype(dt).itemsize].view(dt)
            out[name] = v.reshape(shape).copy() if shape else dt(v[0])
        return out

    @classmethod
    def from_fields(cls, dicts, fingerprint, nq, nv):
        """records packed on the host from one dict of field values per env (missing fields are 0: an idle env with no command or
        program pending); the header is written here"""
        import torch

        lay, R = record_layout(nq, nv), record_size(nq, nv)
        raw = np.zeros((len(dicts), R), np.uint8)
        for i, d in enumerate(dicts):
            unknown = set(d) - set(lay)
            if unknown:
                raise KeyError(f"not record fields: {sorted(unknown)}")
            vals = dict(d, magic=MAGIC, size=R, fingerprint=fingerprint)
            for name, v in vals.items():
                dt, off, shape = lay[name]
                a = np.asarray(v, dtype=dt).reshape(shape)
                raw[i, off:off + a.nbytes] = np.frombuffer(a.tobytes(), np.uint8)
        return cls(torch.from_numpy(raw), nq, nv, fingerprint)

    def to(self, device):
        facade = None
        if self.facade is not None:
            facade = dict(self.facade, observation={k: v.to(device) for k, v in self.facade["observation"].items()}
                          if self.facade.get("observation") is not None else None)
        return EngineState(self.data.to(device), self.nq, self.nv, self.fingerprint, facade)

    def save(self, path):
        import torch

        cpu = self.to("cpu")
        torch.save({"format": "GES1", "nq": self.nq, "nv": self.nv, "fingerprint": self.fingerprint, "data": cpu.data,
                    "facade": cpu.facade}, path)

    @classmethod
    def load(cls, path, device="cpu"):
        import torch

        d = torch.load(path, map_location="cpu", weights_only=True)
        if d.get("format") != "GES1":
            raise ValueError(f"{path}: not an environment state file")
        return cls(d["data"], d["nq"], d["nv"], d["fingerprint"], d.get("facade")).to(device)
