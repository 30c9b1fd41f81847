"""Environment state records (mujoco_rl_ur5_b200/env_state.py, format "GES1" of include/grasp_engine.h) on the host: the model
fingerprint, the record layout of both scenes, packing from field values and the file round trip, and that no per-env row of the
engine is silently left out of a record."""
import os
import re

import numpy as np
import pytest
import torch

from mujoco_rl_ur5_b200.env_state import EXCLUDED, MAGIC, EngineState, fingerprint, record_layout, record_size

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fingerprint_fnv1a_64_vectors():
    assert fingerprint(b"") == 0xCBF29CE484222325
    assert fingerprint(b"a") == 0xAF63DC4C8601EC8C
    assert fingerprint(b"foobar") == 0x85944171F73967E8


@pytest.mark.parametrize("scene, nq, nv, R", [("A", 50, 44, 1536), ("B", 288, 248, 6784)])
def test_record_size_of_both_scenes(scene, nq, nv, R):
    from mujoco_rl_ur5_b200.model.scene import load_scene

    arrays, _ = load_scene(scene)
    assert (int(np.asarray(arrays["nq"]).ravel()[0]), int(np.asarray(arrays["nv"]).ravel()[0])) == (nq, nv)
    assert record_size(nq, nv) == R and R % 128 == 0
    lay = record_layout(nq, nv)
    ends = sorted((off, off + np.dtype(dt).itemsize * int(np.prod(shape, dtype=np.int64))) for dt, off, shape in lay.values())
    assert ends[0][0] == 0 and all(a[1] == b[0] for a, b in zip(ends, ends[1:])), "fields must be packed back to back"
    assert ends[-1][1] <= R < ends[-1][1] + 128
    assert all(off % np.dtype(dt).itemsize == 0 for dt, off, _ in lay.values())


def _fields(rng, nq, nv):
    return {"qpos": rng.standard_normal(nq), "qvel": rng.standard_normal(nv), "qaccws": rng.standard_normal(nv),
            "ctl": rng.standard_normal(32), "cmd_tol": 0.05, "prog_coords": rng.standard_normal(3), "prog_table": 0.91,
            "substeps": 123456789012, "cmd_active": 1, "cmd_mask": 0x1F, "cmd_maxsteps": 1000, "cmd_steps": 17, "cmd_result": 0,
            "prog_phase": 5, "prog_rot": 3, "prog_grasp": 1, "prog_aux": 0x230007, "prog_info": rng.integers(-5, 2000, 12),
            "status": 64, "reward": 1}


def test_from_fields_round_trip():
    rng = np.random.default_rng(0)
    nq, nv, fp = 50, 44, 0x0123456789ABCDEF
    dicts = [_fields(rng, nq, nv) for _ in range(3)]
    s = EngineState.from_fields(dicts, fp, nq, nv)
    assert len(s) == 3 and s.record_bytes == 1536 and s.data.dtype == torch.uint8
    for i, d in enumerate(dicts):
        f = s.fields(i)
        assert f["magic"] == MAGIC and f["size"] == 1536 and int(f["fingerprint"]) == fp
        for k, v in d.items():
            assert np.asarray(f[k]).tobytes() == np.asarray(v, dtype=record_layout(nq, nv)[k][0]).tobytes(), k
    assert torch.equal(s.field("qpos")[1], torch.as_tensor(dicts[1]["qpos"]))
    assert s.field("prog_info").shape == (3, 12) and int(s.field("substeps")[2]) == 123456789012
    assert bytes(s.data[0, :4].numpy()) == b"GES1"
    assert not s.data[:, 1516:].any(), "padding is zero"
    with pytest.raises(KeyError):
        EngineState.from_fields([{"qpos_typo": np.zeros(nq)}], fp, nq, nv)


def test_field_views_write_through():
    s = EngineState.from_fields([{}, {}], 7, 50, 44)
    s.field("qvel")[1, 3] = 2.5
    s.field("prog_phase")[0] = 9
    assert s.fields(1)["qvel"][3] == 2.5 and s.fields(0)["prog_phase"] == 9 and s.fields(1)["prog_phase"] == 0


def test_save_load_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    s = EngineState.from_fields([_fields(rng, 288, 248) for _ in range(2)], 0xFEDCBA9876543210, 288, 248)
    s.facade = {"observation": {"rgb": torch.arange(12, dtype=torch.uint8).reshape(1, 2, 2, 3)}, "step_called": 3, "episode": 2}
    p = str(tmp_path / "state.pt")
    s.save(p)
    t = EngineState.load(p)
    assert (t.nq, t.nv, t.fingerprint) == (288, 248, 0xFEDCBA9876543210)
    assert torch.equal(t.data, s.data)
    assert t.facade["step_called"] == 3 and t.facade["episode"] == 2
    assert torch.equal(t.facade["observation"]["rgb"], s.facade["observation"]["rgb"])
    torch.save({"format": "other"}, p)
    with pytest.raises(ValueError):
        EngineState.load(p)


def test_bad_record_shape_is_refused():
    with pytest.raises(ValueError):
        EngineState(torch.zeros((2, 1535), dtype=torch.uint8), 50, 44, 0)


def test_every_env_row_is_in_the_record_or_excluded():
    """a new per-env row of EnvArrays must be added to the record or to the documented exclusion list"""
    src = open(os.path.join(ROOT, "mujoco_rl_ur5_b200", "csrc", "ge_model.cuh")).read()
    body = re.search(r"struct EnvArrays \{(.*?)\n\};", src, re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    names = set(re.findall(r"\*\s*(\w+)", body))
    assert {"qpos", "qaccws", "ctl", "gws", "ticket", "substeps"} <= names
    in_record = set(record_layout(50, 44)) - {"magic", "size", "fingerprint"}
    assert not (in_record & set(EXCLUDED))
    assert names == in_record | set(EXCLUDED), (sorted(names - in_record - set(EXCLUDED)), sorted((in_record | set(EXCLUDED)) - names))
    hdr = open(os.path.join(ROOT, "include", "grasp_engine.h")).read()
    for k in ("lock", "owed", "done", "ticket", "Hessian overflow rows", "ge_size 13"):
        assert k in hdr, k
