"""Per-stage cycle profile of k_run on the headline workload (GPU).

    tools/build_profile_libs.sh TAG
    python tools/k_run_stage_profile.py exp_libs/libgrasp_engine_TAG_clk.so [exp_libs/libgrasp_engine_TAG_warm.so ...] [--steps K]

Each library runs in a child process (GE_LIB selects it) on bench.py's headline workload: scene A, 4096 envs, chunk 256, grasp
attempts assigned to idle envs with bench's generator seed and draws, `--warmup` untimed steps, then `--steps` profiled ones.  Prints
the cycles per sub-step of every stage (ge_clocks.cuh), summed over all warps and divided by the sub-steps they ran, so the total is
what one warp spends on one sub-step.  A `_warm` library also reports the second, warm pass of the pure stages.  The card name and
power limit are printed first.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = ["PID", "stage_fk", "collision (broad phase, analytic pairs, contact parameters)", "MPR", "stage_rne + stage_crb",
          "smooth forces + mass solve", "stage_constraints", "Newton (warm start, gradient, directions)",
          "Hessian: coupling, lists, islands, offsets", "Hessian: M rows", "Hessian: uncoupled trees", "Hessian: islands", "Cholesky",
          "line search", "nt_update", "Euler", "scheduler / program / load / store", "barrier waits"]
# the slots behind the stages, in ge_clocks.cuh's order
SC_SUBSTEPS, SC_WARM_FK, SC_WARM_RNE_CRB, SC_WARM_MULM, SC_MULM_COLD, SC_HESS_BUILDS, SC_HESS_COUPLED, SC_NUM = range(18, 26)
SLOTS = 4096


def child(lib, steps, warmup):
    os.environ["GE_LIB"] = os.path.abspath(lib)
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    from mujoco_rl_ur5_b200 import engine as engmod
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    L = engmod.load_library()
    fn = L.ge_stage_clocks_warp
    fn.argtypes = [C.c_void_p, C.c_int]
    N, chunk = 4096, 256
    dev = torch.device("cuda", 0)
    env = BatchedGraspEnv(N, "A", 0)
    eng = env.engine
    env.reset()
    gen = torch.Generator(device=dev)
    gen.manual_seed(30000)

    def assign_idle():  # bench.py run_ours
        idle = (eng.busy() == 0)
        u = torch.rand((N, 3), generator=gen, device=dev, dtype=torch.float64)
        coords = torch.stack([-0.2 + 0.4 * u[:, 0], -0.75 + 0.3 * u[:, 1], torch.full((N,), 0.92, device=dev, dtype=torch.float64)], dim=1)
        rot = torch.randint(0, 6, (N,), generator=gen, device=dev, dtype=torch.int32)
        eng.grasp(coords, rot, 0.91, env_mask=idle.to(torch.uint8))

    buf = np.zeros((SLOTS, SC_NUM), dtype=np.uint64)
    for _ in range(warmup):
        assign_idle()
        eng.run_async(chunk)
    torch.cuda.synchronize()
    assert fn(None, 1) == 0, L.ge_last_error()
    ev0, ev1 = torch.cuda.Event(True), torch.cuda.Event(True)
    ms = 0.0
    for _ in range(steps):
        assign_idle()
        ev0.record()
        eng.run_async(chunk)
        ev1.record()
        torch.cuda.synchronize()
        ms += ev0.elapsed_time(ev1)
    assert fn(buf.ctypes.data_as(C.c_void_p), 0) == 0, L.ge_last_error()
    tot = buf.sum(axis=0).astype(np.float64)
    nsub = tot[SC_SUBSTEPS]
    print(json.dumps({"lib": os.path.basename(lib), "substeps": nsub, "kernel_ms": ms, "substeps_per_s": nsub / (ms * 1e-3),
                      "cycles": [float(x) for x in tot]}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.libs[0], a.steps, a.warmup)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card: %s" % card)
    res = []
    for lib in a.libs:
        out = subprocess.run([sys.executable, __file__, lib, "--child", "--steps", str(a.steps), "--warmup", str(a.warmup)],
                             capture_output=True, text=True)
        if out.returncode:
            sys.exit(out.stderr)
        res.append(json.loads(out.stdout.strip().splitlines()[-1]))
    w = max(len(s) for s in STAGES) + 2
    print("cycles per sub-step per warp (profile build: the counters themselves add a little to every stage)")
    print("%-*s" % (w, "stage") + "".join("%14s" % r["lib"].replace("libgrasp_engine_", "").replace(".so", "")[:13] for r in res))
    for r in res:  # the first mul_M of a Newton solve has its own counter (the cold pass of the warm experiment)
        r["rows"] = r["cycles"][:len(STAGES)]
        r["rows"][STAGES.index("Newton (warm start, gradient, directions)")] += r["cycles"][SC_MULM_COLD]
    for i, s in enumerate(STAGES):
        print("%-*s" % (w, s) + "".join("%14.0f" % (r["rows"][i] / r["substeps"]) for r in res))
    print("%-*s" % (w, "total") + "".join("%14.0f" % (sum(r["rows"]) / r["substeps"]) for r in res))
    hess = [STAGES.index(s) for s in STAGES if s.startswith("Hessian")]
    print("%-*s" % (w, "  of which Hessian build") + "".join("%14.0f" % (sum(r["rows"][i] for i in hess) / r["substeps"]) for r in res))
    print("%-*s" % (w, "  of which first mul_M of Newton") + "".join("%14.0f" % (r["cycles"][SC_MULM_COLD] / r["substeps"]) for r in res))
    for name, i in (("warm stage_fk", SC_WARM_FK), ("warm stage_rne + stage_crb", SC_WARM_RNE_CRB), ("warm mul_M", SC_WARM_MULM)):
        if any(r["cycles"][i] for r in res):
            print("%-*s" % (w, name) + "".join("%14.0f" % (r["cycles"][i] / r["substeps"]) for r in res))
    print("%-*s" % (w, "Hessian builds per sub-step") + "".join("%14.3f" % (r["cycles"][SC_HESS_BUILDS] / r["substeps"]) for r in res))
    print("%-*s" % (w, "  share with a coupled tree") + "".join("%14.3f" % (r["cycles"][SC_HESS_COUPLED] / max(r["cycles"][SC_HESS_BUILDS], 1))
                                                                 for r in res))
    print("%-*s" % (w, "sub-steps / s (profile build)") + "".join("%14.0f" % r["substeps_per_s"] for r in res))


if __name__ == "__main__":
    main()
