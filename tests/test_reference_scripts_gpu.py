"""Acceptance run of the reference's UNCHANGED scripts against the H100 engine (north star: "... so Grasping_Agent_multidiscrete.py
runs unchanged against it"; VERDICT r01 row N2).

`example_agent.py` (reference: example_agent.py:8-26) and `Grasping_Agent_multidiscrete.main` (:515-583) are executed from the
staged byte-for-byte copies in baseline/_ref (tools/stage_reference.py; /root/reference when it exists) with
mujoco_rl_ur5_b200/compat first on PYTHONPATH, so `gym.make("gym_grasper:Grasper-v0", ...)` builds the CUDA-backed GraspEnv on
the reference's default 40-object scene.  Loops are shortened from outside (tests/run_reference_script.py): 1 episode x 3 steps.
Checked: exit code 0, the script reaches its own last line, three rewards in {0, 1}, default scene = many_objects (B), TensorBoard
event file / checkpoint written by the agent's own code.
"""
import glob
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPAT = os.path.join(ROOT, "mujoco_rl_ur5_b200", "compat")
CANDIDATES = [os.environ.get("GRASP_REFERENCE_DIR", ""), os.path.join(ROOT, "baseline", "_ref"), "/root/reference"]


def _ref_dir():
    for d in CANDIDATES:
        if d and os.path.exists(os.path.join(d, "Grasping_Agent_multidiscrete.py")) and os.path.exists(os.path.join(d, "example_agent.py")):
            return d
    return None


def _run(which, tmp_path, timeout, oracle_backed=False):
    ref = _ref_dir()
    if ref is None:
        pytest.skip("reference scripts not staged: run tools/stage_reference.py where /root/reference exists")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, COMPAT, ref])
    env.pop("GRASP_SCENE", None)
    if oracle_backed:  # CPU dry run: oracle behind the façade, 6-object scene (the oracle does ~100 sub-steps/s on the 40-object one)
        env["GRASP_TEST_ENGINE"], env["GRASP_SCENE"], env["CUDA_VISIBLE_DEVICES"] = "oracle", "A", ""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "run_reference_script.py"), which, ref, "1", "3"], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert "__SCRIPT_DONE__" in r.stdout
    rewards = [line.split() for line in r.stdout.splitlines() if line.startswith("REWARD ")]
    assert len(rewards) == 3 and all(w[1] in ("0", "1") for w in rewards), rewards
    assert all(w[3] == ("A" if oracle_backed else "B") for w in rewards)  # GPU run: the reference's default scene (GraspingEnv.py:30)
    return r.stdout


def test_staging_tool_lists_the_scripts_the_test_needs():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import stage_reference

    assert {"example_agent.py", "Grasping_Agent_multidiscrete.py", "Modules.py"} <= set(stage_reference.FILES)


@pytest.mark.gpu
def test_example_agent_runs_unchanged(tmp_path):
    out = _run("example", tmp_path, 900)
    assert "Finished." in out                      # example_agent.py:31
    assert "Model timestep:" in out                # env.print_info() (example_agent.py:13)
    assert out.count("EPISODE 1 STEP") == 3


@pytest.mark.gpu
def test_grasping_agent_main_runs_unchanged(tmp_path):
    out = _run("agent", tmp_path, 1200)
    assert "Finished training (rand_seed = 999)." in out          # Grasping_Agent_multidiscrete.py:580
    assert out.count("Filling the replay buffer ...") == 3        # learn() before 2 * BATCH_SIZE transitions (:396-398)
    assert glob.glob(os.path.join(str(tmp_path), "runs", "*", "events.out.tfevents.*"))   # the agent's own SummaryWriter
    assert glob.glob(os.path.join(str(tmp_path), "*_weights.pt"))                          # SAVE_WEIGHTS checkpoint (:563-577)


def test_reference_scripts_run_on_the_oracle_backed_facade(tmp_path):
    """CPU: the same two scripts with the CPU oracle behind the façade (tests/oracle_engine.py) - covers the host-side mirror of the
    reference interface (gym shim, GraspEnv, MJ_Controller, result strings, observation dict) without a GPU"""
    out = _run("example", tmp_path, 600, oracle_backed=True)
    assert "Finished." in out and "GRASP_SCENE=A overrides" in out
    out = _run("agent", tmp_path, 900, oracle_backed=True)
    assert "Finished training (rand_seed = 999)." in out
