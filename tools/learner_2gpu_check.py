"""Multi-GPU learner check (run under torchrun, one rank per GPU):
every rank takes its own batch through QNetLearner.learn_step with the per-group gradient all-reduce; afterwards (a) the parameters are
bit-identical on all ranks and (b) they equal, to fp32 reduction-order noise, what ONE process gets by averaging the per-batch gradients
itself and applying the same optimizer step.  Prints one JSON line on rank 0.  --optimizer sgd / --accumulate K check SGD and gradient
accumulation: every rank then takes K micro-batches, and the single process sums each rank's K micro-batch gradients (loss / K) before it
averages over the ranks.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 tools/learner_2gpu_check.py
      [--optimizer sgd] [--accumulate 2]
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mujoco_rl_ur5_b200.qnet_learn import QNetLearner  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
ap = argparse.ArgumentParser()
ap.add_argument("--optimizer", choices=("adam", "sgd"), default="adam")
ap.add_argument("--accumulate", type=int, default=1)
args = ap.parse_args()
K = args.accumulate
B = 3 * K


def batch(r):
    g = torch.Generator().manual_seed(100 + r)
    return (torch.rand(B, 4, 200, 200, generator=g), torch.randint(0, 6 * 200 * 200, (B, 1), generator=g), (torch.rand(B, 1, generator=g) < 0.5).float())


L = QNetLearner(seed=0, device=local, process_group=dist.group.WORLD, optimizer=args.optimizer, accumulate=K)
loss = L.learn_step(*[x.cuda() for x in batch(rank)])
torch.cuda.synchronize()
mine = L.flat.clone()
ref0 = mine.clone()
dist.broadcast(ref0, 0)
same = bool(torch.equal(mine, ref0))
flags = [None] * world
dist.all_gather_object(flags, same)
out = {"world": world, "optimizer": args.optimizer, "accumulate": K, "loss_rank0": loss, "params_identical_on_all_ranks": all(flags)}
if rank == 0:
    # single process: every rank's K micro-batch gradients (loss / K each) summed, then averaged over the ranks by hand, same optimizer step
    S = QNetLearner(seed=0, device=local, optimizer=args.optimizer)
    acc = torch.zeros_like(S.grad)
    for r in range(world):
        st, ac, rw = [x.cuda() for x in batch(r)]
        for k in range(K):
            rows = slice(3 * k, 3 * (k + 1))
            q, saved = S.forward_train(st[rows])
            S.backward(q, saved, ac[rows], rw[rows], weight=None if K == 1 else torch.full((3,), 1.0 / K, device="cuda"))
            acc += S.grad
    S.grad.copy_(acc / world)
    S.step_count += 1
    S._optimizer_step(S.grad)
    torch.cuda.synchronize()
    # Adam's first step moves every weight by ~lr * sign(g) (SGD's by lr * g): compare the updates, allowing sign flips only where |g| is at
    # rounding level
    d = (S.flat - mine).abs()
    out["max_abs_param_diff_vs_single_process"] = float(d.max())
    out["fraction_of_params_differing_by_more_than_1e-5"] = float((d > 1e-5).float().mean())
    out["ok"] = bool(out["params_identical_on_all_ranks"] and out["fraction_of_params_differing_by_more_than_1e-5"] < 0.01)
    print(json.dumps(out), flush=True)
dist.barrier()
dist.destroy_process_group()
