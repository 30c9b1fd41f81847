#!/usr/bin/env python
"""Runner used by tests/test_reference_scripts_gpu.py: executes one of the reference's OWN scripts, byte for byte as staged in
baseline/_ref (or /root/reference), against the H100 engine.  Only loop lengths are shortened, from the OUTSIDE:

  example  : example_agent.py (reference: example_agent.py:1-31) has module-level `N_EPISODES = 100` / `N_STEPS = 100`; its source
             text is read, those two literals are replaced IN MEMORY and the result is exec'd (the file is not touched).
  agent    : `import Grasping_Agent_multidiscrete as G`, set G.N_EPISODES / G.STEPS_PER_EPISODE (module globals read by main() at call
             time, Grasping_Agent_multidiscrete.py:515-583), call G.main().

The façade's `GraspEnv.step` is wrapped to print every reward as `REWARD <r>` so the test can check them; nothing else of
the product is patched.  argv: <example|agent> <reference dir> <episodes> <steps>
"""
import os
import sys


def main():
    which, ref, episodes, steps = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
    from mujoco_rl_ur5_b200 import grasp_env

    orig = grasp_env.GraspEnv.step

    def step(self, action, *a, **k):
        out = orig(self, action, *a, **k)
        print("REWARD", int(out[1]), "SCENE", self.scene, flush=True)
        return out

    grasp_env.GraspEnv.step = step
    if os.environ.get("GRASP_TEST_ENGINE") == "oracle":
        # CPU dry run of the host-side façade (the `-m "not gpu"` suite): the engine behind GraspEnv is the CPU oracle wrapped in the
        # BatchedEngine surface (tests/oracle_engine.py) - test infrastructure, the product itself has no CPU path
        from mujoco_rl_ur5_b200 import controller
        from tests.oracle_engine import OracleEngine

        grasp_env.BatchedEngine = controller.BatchedEngine = OracleEngine
    if which == "example":
        src = open(os.path.join(ref, "example_agent.py")).read()
        assert "N_EPISODES = 100" in src and "N_STEPS = 100" in src
        src = src.replace("N_EPISODES = 100", "N_EPISODES = %d" % episodes).replace("N_STEPS = 100", "N_STEPS = %d" % steps)
        exec(compile(src, os.path.join(ref, "example_agent.py"), "exec"), {"__name__": "__main__"})
    else:
        import Grasping_Agent_multidiscrete as G

        assert os.path.dirname(os.path.abspath(G.__file__)) == os.path.abspath(ref)
        G.N_EPISODES, G.STEPS_PER_EPISODE = episodes, steps
        G.main()
    print("__SCRIPT_DONE__", flush=True)


if __name__ == "__main__":
    main()
