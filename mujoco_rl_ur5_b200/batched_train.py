"""BatchedTrainer: the reference's online training loop (Grasping_Agent_multidiscrete.main, :515-583) over N device environments.

Per transition the reference runs  transform_observation -> epsilon_greedy -> env.step -> memory.push -> learn().  Here one batched step
does that for N envs at once, every part a kernel of this project:
    gq_obs_to_state_keyed (acting state = the state that is stored) -> QNetForward with per-image BatchNorm on the learner's current
    weights, in chunks -> gq_argmax -> gq_sample_actions (epsilon-greedy, depth-filtered random actions) -> BatchedGraspEnv.step ->
    ObservationReplay.push_batch -> `updates_per_step` x QNetLearner.learn_step on ObservationReplay.sample(batch_size).
Every random choice (depth noise, ColorJitter, the epsilon draw, the random-action candidates) is keyed on (seed, global env index,
step), so the actions and states of an env do not depend on how the envs are batched or sharded over GPUs.

Transition numbers: env g (global index) of batched step t takes number n = steps_done + t * N_total + g, where steps_done is the count
at the start or the resume; its epsilon is EPS_END + (EPS_START - EPS_END) exp(-n / EPS_DECAY) as in epsilon_greedy (:244-246), and
its keyed step counter is the number of the batch's first transition.  Checkpoints are the reference's main() dict (:560-572).

Cost: updates_per_step defaults to n_envs, the reference's one learn() per transition.  A learn() step of batch 12 is a forward and
backward of the whole network, so at that ratio the learner dominates a batched step; DESIGN.md section 5 gives measured times.

Prioritized replay (`prioritized=dict(alpha, beta0, beta_updates, eps)`, off by default): the replay is a
PrioritizedObservationReplay, every update draws its batch in proportion to the priorities, keyed on (seed, learner update, rank),
trains on the importance-weighted loss with beta going linearly from beta0 to 1 over beta_updates updates, and writes the batch's new
priorities (|r - q_pred| + eps)^alpha back.  Without it the trainer is the reference's uniform rule, unchanged.

Bootstrapped Q-learning (`gamma` > 0, the reference's GAMMA branch of learn(), :105-115,140-144,410-413,430-437; default gamma = 0, the
branch the reference runs): the replay also keeps each transition's next observation, keyed on the next batched step (key + N_total),
so that its regenerated state is bit for bit the state the env acts on next; an episode's last transition bootstraps from the
observation before the reset, as the reference does.  Before learner update u the target network (the learner's eval-mode,
BatchNorm-folded forward) is rebuilt when u % target_update == 0 and after a construction or resume, and every update trains on
y = min(1, r + gamma * max_a' Q_target(s', a')) (fp32; gq_head_max_target), which keeps y in binary_cross_entropy's [0, 1] (a successful
grasp ends the bootstrapped return) and is r at gamma = 0.  With prioritized replay the priorities are |y - q_pred|.

Optimiser and accumulation (`optimizer`, `momentum`, `accumulate`; the reference's OPTIMIZER and NUMBER_ACCUMULATIONS_BEFORE_UPDATE):
Adam by default, or SGD with momentum; a loaded checkpoint brings its own.  With accumulate = K one update draws batch_size * K
transitions in one call (the reference's BATCH_SIZE = MAX_POSSIBLE_SAMPLES * K; with prioritized replay K * batch_size strata whose
importance weights are normalised over the whole draw), QNetLearner.learn_step trains on them as K micro-batches of batch_size with one
optimizer step, and updating starts once the replay holds 2 * batch_size * K transitions.  At gamma > 0 the targets of all the drawn
next states come from the one target network before the step.  `updates` in the per-step record counts optimizer steps.

Standardised observations (`standardize` = a `mean_and_std` path or its 8 values; the reference's transform_observation(normalize=False),
:311-354): the acting states, the replay's regenerated states (next states at gamma > 0 included) and so the epsilon-greedy arg-max use
gq_obs_to_state_standard under the same (seed, env, step) keys, with the depth noise noise_std in standardised units and no ColorJitter;
gq_sample_actions still reads the raw depth.  The checkpoint gains "mean_and_std"; a resume from such a checkpoint uses its values, and
passing different ones is an error.  Without it every state, the replay and the checkpoint are the min-max path's.

Multi-GPU (torchrun): rank r runs envs [r N, (r + 1) N) of N_total = world N, the learner all-reduces its gradients over the process
group, each rank keeps its own replay and sampling stream random.Random(seed + rank), the counters are summed when a checkpoint is
written and rank 0 writes it.
"""
import argparse
import json
import math
import random
import sys
from collections import defaultdict

import numpy as np

from .batched_env import BatchedGraspEnv
from .qnet_learn import QNetLearner, check_optimizer
from .replay_buffer import ObservationReplay, PrioritizedObservationReplay

EPS_START, EPS_END, EPS_DECAY = 1.0, 0.2, 8000   # Grasping_Agent_multidiscrete.py:35-37
COUNTERS = ("greedy_rotations", "greedy_rotations_successes", "random_rotations_successes")
PER_DEFAULTS = dict(alpha=0.6, beta0=0.4, eps=1e-6)  # Schaul et al. 2016, proportional variant; beta_updates has no default


def per_beta(update, beta0, beta_updates):
    """importance-sampling exponent of learner update `update` (0-based): linear from beta0 at update 0 to 1 at beta_updates, then 1"""
    if beta_updates <= 0:
        return 1.0
    return beta0 + (1.0 - beta0) * min(1.0, update / beta_updates)


def check_bootstrap(gamma, target_update):
    """-> (gamma as a float, target_update); ValueError unless 0 <= gamma <= 1 and target_update is a positive int when gamma > 0 and
    None when gamma = 0 (there is no target network then)"""
    if isinstance(gamma, bool) or not isinstance(gamma, (int, float)) or not 0.0 <= float(gamma) <= 1.0:
        raise ValueError(f"gamma must be a number in [0, 1], not {gamma!r}")
    gamma = float(gamma)
    if gamma > 0.0:
        if isinstance(target_update, bool) or not isinstance(target_update, int) or target_update < 1:
            raise ValueError(f"gamma > 0 needs target_update, a positive int (learner updates between target network syncs), not {target_update!r}")
    elif target_update is not None:
        raise ValueError(f"target_update is for gamma > 0 (there is no target network at gamma = 0); got {target_update!r}")
    return gamma, target_update


def epsilon(n, eps_start=EPS_START, eps_end=EPS_END, eps_decay=EPS_DECAY):
    """the reference's exploration rate of transition n (epsilon_greedy, :244-246), with its arithmetic (math.exp of -1.0 n / decay)"""
    return eps_end + (eps_start - eps_end) * math.exp(-1.0 * n / eps_decay)


def resolve_standardize(standardize, ckpt=None):
    """-> the 8 statistics (obs_stats types) of the standardised transform, or None: `standardize` is None, a `mean_and_std` path or the
    8 values; a checkpoint's "mean_and_std" is used when `standardize` is None and must equal it otherwise (ValueError)"""
    from .obs_stats import check_mean_and_std, load_mean_and_std

    if isinstance(standardize, (str, bytes)) or hasattr(standardize, "__fspath__"):
        standardize = load_mean_and_std(standardize)
    elif standardize is not None:
        standardize = check_mean_and_std(standardize)
    stored = None if not ckpt or ckpt.get("mean_and_std") is None else check_mean_and_std(ckpt["mean_and_std"])
    if stored is not None and standardize is not None and [float(v) for v in stored] != [float(v) for v in standardize]:
        raise ValueError(f"the checkpoint was trained on standardised observations with mean_and_std {[float(v) for v in stored]}, "
                         f"not {[float(v) for v in standardize]}")
    return stored if standardize is None else standardize


def load_checkpoint(path_or_dict):
    import torch

    if isinstance(path_or_dict, dict):
        return path_or_dict
    return torch.load(path_or_dict, map_location="cpu", weights_only=False)


class BatchedTrainer:
    def __init__(self, n_envs, scene="A", device=0, seed=0, batch_size=12, mem_size=None, updates_per_step=None, lr=1e-3, eps_start=EPS_START,
                 eps_end=EPS_END, eps_decay=EPS_DECAY, load=None, env_index_offset=None, n_total=None, process_group=None, chunk=64, max_draws=256,
                 noise_std=0.001, log=None, prioritized=None, gamma=0.0, target_update=None, optimizer=None, momentum=0.9, accumulate=1,
                 standardize=None):
        import torch
        import torch.distributed as dist

        self.gamma, self.target_update = check_bootstrap(gamma, target_update)
        _, self.accumulate, momentum = check_optimizer("adam" if optimizer is None else optimizer, accumulate, momentum)
        ckpt = None if load is None else load_checkpoint(load)
        self.standardize = resolve_standardize(standardize, ckpt)
        self.torch = torch
        self.pg = process_group
        rank, world = (dist.get_rank(process_group), dist.get_world_size(process_group)) if process_group is not None else (0, 1)
        self.rank = rank
        self.n_envs = int(n_envs)
        self.env_offset = rank * self.n_envs if env_index_offset is None else int(env_index_offset)
        self.n_total = world * self.n_envs if n_total is None else int(n_total)
        self.env = BatchedGraspEnv(self.n_envs, scene, device, env_index_offset=self.env_offset)
        self.dev = self.env.engine.device
        self.seed = int(seed)
        self.batch_size = int(batch_size)
        self.updates_per_step = self.n_envs if updates_per_step is None else int(updates_per_step)
        self.eps_start, self.eps_end, self.eps_decay = eps_start, eps_end, eps_decay
        self.chunk, self.max_draws, self.noise_std = int(chunk), int(max_draws), float(noise_std)
        self.log = log
        opt = {} if optimizer is None else {"optimizer": optimizer}
        if ckpt is None:
            self.learner = QNetLearner(None, device, lr=lr, seed=self.seed, process_group=process_group, momentum=momentum, accumulate=self.accumulate,
                                       **opt)
        else:  # as the reference's constructor: the optimizer state (and with it the optimizer, learning rate and momentum) comes from the
            # checkpoint (:157-179); an explicit optimizer must be the checkpoint's
            self.learner = QNetLearner.from_checkpoint(ckpt, device, process_group=process_group, accumulate=self.accumulate, **opt)
        ckpt = ckpt or {}
        self.steps_done = int(ckpt.get("step", 0))
        # as the reference (:161-163, :182): EPS_START for a fresh agent, the checkpoint's value or EPS_STEADY = 0 for a loaded one
        self.eps_threshold = float(ckpt.get("epsilon", 0.0)) if ckpt else float(eps_start)
        # counters restored from the checkpoint (the same on every rank) and counted in this run (summed over the ranks when saved)
        self.base_counters = {k: defaultdict(int, {str(r): int(v) for r, v in (ckpt.get(k) or {}).items()}) for k in COUNTERS}
        self.run_counts = np.zeros((len(COUNTERS), len(self.env.rotations)), dtype=np.int64)
        mem = max(2000, 4 * self.n_envs) if mem_size is None else int(mem_size)
        W, H = self.env.IMAGE_WIDTH, self.env.IMAGE_HEIGHT
        self.per = None
        nxt = {"next_obs": True} if self.gamma > 0 else {}  # at gamma = 0 the replays are built exactly as without bootstrapping
        if self.standardize is not None:
            nxt["standardize"] = self.standardize
        if prioritized is None:
            self.replay = ObservationReplay(mem, (H, W), device=self.dev, rng=random.Random(self.seed + rank), **nxt)
        else:
            unknown = set(prioritized) - set(PER_DEFAULTS) - {"beta_updates"}
            if unknown or "beta_updates" not in prioritized:
                raise ValueError(f"prioritized takes alpha, beta0, beta_updates (required) and eps; got {sorted(prioritized)}")
            self.per = {**PER_DEFAULTS, **prioritized}
            self.replay = PrioritizedObservationReplay(mem, (H, W), device=self.dev, alpha=self.per["alpha"], eps=self.per["eps"], **nxt)
        A = self.env.arrays
        cam = self.env.cam
        self.camera = (float(np.asarray(A["cam_fovy"]).ravel()[cam]), np.asarray(A["cam_pos0"], dtype=np.float64).reshape(-1, 3)[cam],
                       np.asarray(A["cam_mat0"], dtype=np.float64).reshape(-1, 9)[cam])
        self.z_min = self.env.TABLE_HEIGHT - 0.01                               # :275
        self.depth_threshold = float(np.round(self.camera[1][2] - self.env.TABLE_HEIGHT + 0.01, 3))  # :130-135
        self.genv = self.env_offset + torch.arange(self.n_envs, dtype=torch.int64, device=self.dev)
        self.batched_steps = 0

    # ------------------------------------------------------------------ acting
    def acting_states(self, obs, step):
        """the keyed training transform of the observation: what the agent acts on and what the replay regenerates"""
        t = self.torch
        if self.standardize is not None:
            return self.learner.fw.obs_to_state_standard(obs, self.standardize, self.depth_threshold, self.noise_std, self.seed, step, self.genv)
        return self.learner.fw.obs_to_state_keyed(obs["rgb"], obs["depth"], self.genv, t.full((self.n_envs,), step, dtype=t.int64, device=self.dev),
                                                  self.seed, depth_threshold=self.depth_threshold, noise_std=self.noise_std)

    def greedy_indices(self, states):
        """flat arg-max rot*H*W + y*W + x per image, forward and arg-max chunk by chunk (the Q-maps of all envs are never held at once)"""
        t = self.torch
        fw = self.learner.fw
        idx = t.empty(states.shape[0], dtype=t.int32, device=self.dev)
        val = t.empty(states.shape[0], dtype=t.float32, device=self.dev)
        for i in range(0, states.shape[0], self.chunk):
            q = fw.forward(states[i:i + self.chunk])
            fw._ck(fw.L.gq_argmax(fw._p(q), q.shape[0], q[0].numel(), fw._p(idx[i:]), fw._p(val[i:]), fw._stream()), "gq_argmax")
        return idx

    def epsilons(self):
        """epsilon of every env's transition in the current batched step"""
        base = self.steps_done + self.env_offset
        return [epsilon(base + i, self.eps_start, self.eps_end, self.eps_decay) for i in range(self.n_envs)]

    def act(self, obs):
        """-> (acting states, actions [N,2] int32, is_random [N] bool, exhausted [N] bool) for the current batched step"""
        t = self.torch
        step = self.steps_done & 0xFFFFFFFF
        states = self.acting_states(obs, step)
        idx = self.greedy_indices(states)
        eps = t.tensor(self.epsilons(), dtype=t.float64)
        act, rnd, exh = self.learner.fw.sample_actions(obs["depth"], idx, eps, self.genv, step, self.seed, self.camera, self.z_min,
                                                       len(self.env.rotations), self.max_draws)
        return states, act, rnd, exh

    # ------------------------------------------------------------------ one batched step
    def step(self, mark=None):
        """one batched step; `mark(name)` (optional) is called after each phase - "act", "env_step", "push", "learn" - and before the first
        with "start" (tools/train_profile.py records a CUDA event there)"""
        t = self.torch
        mark = mark or (lambda name: None)
        env = self.env
        obs = env.current_observation
        key = self.steps_done & 0xFFFFFFFF
        mark("start")
        _, act, rnd, exh = self.act(obs)
        mark("act")
        next_obs, reward, _, _ = env.step(act)
        mark("env_step")
        HW = env.IMAGE_WIDTH * env.IMAGE_HEIGHT
        flat = act[:, 1].to(t.int64) * HW + act[:, 0].to(t.int64)
        nxt = {}
        if self.gamma > 0:  # the next observation under the key the next batched step acts with
            nxt = dict(next_rgb=next_obs["rgb"], next_depth=next_obs["depth"],
                       next_steps=t.full((self.n_envs,), (self.steps_done + self.n_total) & 0xFFFFFFFF, dtype=t.int64))
        self.replay.push_batch(obs["rgb"], obs["depth"], flat, t.from_numpy(reward.astype(np.float32)), self.genv,
                               t.full((self.n_envs,), key, dtype=t.int64), **nxt)
        mark("push")
        losses = []
        if len(self.replay) >= 2 * self.batch_size * self.accumulate:  # :396-399, BATCH_SIZE = MAX_POSSIBLE_SAMPLES * accumulations
            for _ in range(self.updates_per_step):
                losses.append(self.update())
        mark("learn")
        # update_tensorboard's counters (:448-466), keyed by str(rotation) like the reference's defaultdicts
        rot = act[:, 1].cpu().numpy()
        rnd_h, exh_h = rnd.cpu().numpy(), exh.cpu().numpy()
        ok = reward == 1
        R = len(env.rotations)
        self.run_counts[0] += np.bincount(rot[~rnd_h], minlength=R)[:R]
        self.run_counts[1] += np.bincount(rot[~rnd_h & ok], minlength=R)[:R]
        self.run_counts[2] += np.bincount(rot[rnd_h & ok], minlength=R)[:R]
        self.steps_done += self.n_total
        self.eps_threshold = epsilon(self.steps_done - 1, self.eps_start, self.eps_end, self.eps_decay)  # the last transition's, as the reference keeps it
        self.batched_steps += 1
        self.last_step = {"actions": act.cpu().numpy(), "is_random": rnd_h, "exhausted": exh_h, "reward": reward}
        mean = lambda m: float(reward[m].mean()) if m.any() else None
        rec = {"rank": self.rank, "step": self.batched_steps, "steps_done": self.steps_done, "epsilon": self.eps_threshold, "n_greedy": int((~rnd_h).sum()),
               "n_random": int(rnd_h.sum()), "n_exhausted": int(exh_h.sum()), "mean_reward_greedy": mean(~rnd_h), "mean_reward_random": mean(rnd_h),
               "updates": len(losses), "mean_loss": float(np.mean(losses)) if losses else None}
        if self.log is not None:
            self.log.write(json.dumps(rec) + "\n")
            self.log.flush()
        return rec

    def update(self):
        """one learner update (the reference's learn()) on a batch of batch_size * accumulate transitions drawn from the replay in one
        call -> its loss"""
        if self.per is not None:
            return self.prioritized_update()
        n = self.batch_size * self.accumulate
        if self.gamma > 0:
            s, a, r, s2 = self.replay.sample(n, self.learner.fw, self.seed, self.depth_threshold, self.noise_std)
            return self.learner.learn_step(s, a, self.bellman_targets(s2, r))
        s, a, r = self.replay.sample(n, self.learner.fw, self.seed, self.depth_threshold, self.noise_std)
        return self.learner.learn_step(s, a, r)

    def prioritized_update(self):
        """one learner update on a prioritized batch: draw (keyed on the learner's update count and this rank), weighted learn step,
        new priorities of the drawn slots.  -> the weighted loss"""
        u = self.learner.step_count
        beta = per_beta(u, self.per["beta0"], self.per["beta_updates"])
        out = self.replay.sample(self.batch_size * self.accumulate, self.learner.fw, self.seed, beta, u, self.rank, self.depth_threshold, self.noise_std)
        if self.gamma > 0:
            s, a, r, s2, idx, w = out
            r = self.bellman_targets(s2, r)
        else:
            s, a, r, idx, w = out
        loss, qsel = self.learner.learn_step(s, a, r, return_pred=True, weight=w)
        self.replay.update_priorities(idx, qsel, r)
        return loss

    def bellman_targets(self, next_states, reward):
        """y [B] f32 = min(1, r + gamma max_a' Q_target(s', a')) for the coming learner update; first rebuilds the target network from
        the learner when it has none yet (a fresh or resumed trainer) or the update count is a multiple of target_update"""
        L = self.learner
        if L.target is None or L.step_count % self.target_update == 0:
            L.sync_target()
        return L.target.max_target(next_states, reward, self.gamma)[1]

    def train(self, episodes, steps_per_episode):
        for _ in range(episodes):
            self.env.reset()
            for _ in range(steps_per_episode):
                self.step()

    # ------------------------------------------------------------------ checkpoints
    def counters(self):
        """the three rotation counters (dicts str(rot) -> count) of the reference, this run's counts summed over the ranks"""
        t = self.torch
        counts = self.run_counts
        if self.pg is not None:
            import torch.distributed as dist

            c = t.from_numpy(counts).to(self.dev)
            dist.all_reduce(c, op=dist.ReduceOp.SUM, group=self.pg)
            counts = c.cpu().numpy()
        out = {}
        for i, k in enumerate(COUNTERS):
            d = defaultdict(int, self.base_counters[k])
            for r in range(counts.shape[1]):
                if counts[i, r]:
                    d[str(r)] += int(counts[i, r])
            out[k] = d
        return out

    def checkpoint(self):
        """the dict the reference's main() saves (:560-572); with SGD also the learner's "learner_step" (QNetLearner.checkpoint), with
        standardised observations also "mean_and_std" (8 Python floats: the checkpoint holds no numpy objects)"""
        ck = self.learner.checkpoint()
        extra = {"learner_step": ck["learner_step"]} if "learner_step" in ck else {}
        stats = getattr(self, "standardize", None)  # absent on objects that only carry the checkpoint's fields
        if stats is not None:
            extra["mean_and_std"] = [float(v) for v in stats]
        return {"step": self.steps_done, "model_state_dict": ck["model_state_dict"], "optimizer_state_dict": ck["optimizer_state_dict"],
                "epsilon": self.eps_threshold, **self.counters(), **extra}

    def save(self, path):
        """writes the checkpoint from rank 0 (every rank must call it: the counters are summed over the ranks)"""
        ck = self.checkpoint()
        if self.rank == 0:
            self.torch.save(ck, path)
        return ck

    def close(self):
        self.env.close()


def main(argv=None):
    p = argparse.ArgumentParser(prog="python -m mujoco_rl_ur5_b200.batched_train", description=__doc__.split("\n")[0])
    p.add_argument("--envs", type=int, default=256, help="environments per GPU")
    p.add_argument("--scene", default="A")
    p.add_argument("--episodes", type=int, default=1)
    p.add_argument("--steps-per-episode", type=int, default=50)
    p.add_argument("--updates-per-step", type=int, default=None, help="learn() calls per batched step (default: --envs, one per transition)")
    p.add_argument("--batch-size", type=int, default=12, help="transitions per forward/backward (the reference's MAX_POSSIBLE_SAMPLES)")
    p.add_argument("--mem-size", type=int, default=None, help="replay capacity per GPU (default: max(2000, 4 envs))")
    p.add_argument("--lr", type=float, default=1e-3)
    p.add_argument("--eps-start", type=float, default=EPS_START)
    p.add_argument("--eps-end", type=float, default=EPS_END)
    p.add_argument("--eps-decay", type=float, default=EPS_DECAY)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--load", default=None, help="checkpoint to resume from (the reference's or this trainer's)")
    p.add_argument("--out", default=None, help="checkpoint written at the end")
    p.add_argument("--prioritized", action="store_true", help="prioritized experience replay (proportional); beta reaches 1 after the number of updates this run plans")
    p.add_argument("--per-alpha", type=float, default=PER_DEFAULTS["alpha"], help="priority exponent (with --prioritized)")
    p.add_argument("--per-beta0", type=float, default=PER_DEFAULTS["beta0"], help="initial importance-sampling exponent (with --prioritized)")
    p.add_argument("--gamma", type=float, default=0.0, help="discount of the bootstrapped target r + gamma max Q_target(s') (0: the reward alone)")
    p.add_argument("--target-update", type=int, default=None, help="learner updates between target network syncs (required with --gamma > 0)")
    p.add_argument("--optimizer", choices=("adam", "sgd"), default=None, help="adam, or sgd with momentum (default: the --load checkpoint's, else adam)")
    p.add_argument("--momentum", type=float, default=0.9, help="SGD momentum of a fresh run (a loaded checkpoint keeps its own)")
    p.add_argument("--accumulate", type=int, default=1,
                   help="micro-batches of --batch-size per optimizer step, gradients summed (the reference's NUMBER_ACCUMULATIONS_BEFORE_UPDATE)")
    p.add_argument("--standardize", default=None, metavar="PATH",
                   help="a mean_and_std file (python -m mujoco_rl_ur5_b200.normalize): act and learn on standardised observations")
    a = p.parse_args(argv)
    try:
        check_bootstrap(a.gamma, a.target_update)
        check_optimizer(a.optimizer or "adam", a.accumulate, a.momentum)
        if a.standardize is not None:
            resolve_standardize(a.standardize)
    except OSError as e:
        p.error(f"--standardize: {e}")
    except ValueError as e:
        p.error(str(e))
    import os

    import torch
    import torch.distributed as dist

    pg, device = None, 0
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:  # torchrun
        device = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(device)
        dist.init_process_group("nccl")
        pg = dist.group.WORLD
    per = None
    if a.prioritized:
        planned = a.episodes * a.steps_per_episode * (a.envs if a.updates_per_step is None else a.updates_per_step)
        per = dict(alpha=a.per_alpha, beta0=a.per_beta0, beta_updates=planned)
    tr = BatchedTrainer(a.envs, a.scene, device, seed=a.seed, batch_size=a.batch_size, mem_size=a.mem_size, updates_per_step=a.updates_per_step, lr=a.lr,
                        eps_start=a.eps_start, eps_end=a.eps_end, eps_decay=a.eps_decay, load=a.load, process_group=pg,
                        log=sys.stdout if (pg is None or dist.get_rank() == 0) else None, prioritized=per, gamma=a.gamma,
                        target_update=a.target_update, optimizer=a.optimizer, momentum=a.momentum, accumulate=a.accumulate, standardize=a.standardize)
    try:
        tr.train(a.episodes, a.steps_per_episode)
        if a.out:
            tr.save(a.out)
    finally:
        tr.close()
        if pg is not None:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
