"""Device-resident replay buffer with the reference's sampling semantics (SURVEY 8f.2, first half of the learner).

Reference: `Modules.ReplayBuffer` (Modules.py:28-55) — a Python list of `simple_Transition(state, action, reward)` used as a
ring (`position` wraps at `size`), `random.seed(20)` at construction, and
    sample(B) = random.sample(memory, B - 1) + [memory[position - 1]]       (uniform without replacement + the newest)
The agent pushes one transition per env step (Grasping_Agent_multidiscrete.py:552) and samples BATCH_SIZE = 12 in `learn()`
(:401) once the buffer holds 2 * BATCH_SIZE.

Here the transitions live in preallocated tensors on one device (states [size,4,H,W], flat actions, rewards), a batched
environment pushes N transitions at once, and `sample` draws the SAME indices the reference would: `random.sample` picks
positions through `randbelow` only, so sampling `range(len)` with the same generator state returns the indices of the
elements the reference's list sampling returns.  By default the generator is Python's global `random` module seeded with
20 exactly like the reference (the unchanged agent draws its epsilon from the same stream); pass `rng=random.Random(20)` for
a private stream (a generator passed in is used as it is, never re-seeded).  DeviceReplayBuffer's storage and gathers are tensor plumbing
(any torch device); ObservationReplay, the online trainer's memory, stores observations and regenerates states with a kernel.
PrioritizedObservationReplay replaces the uniform draw with prioritized replay (Schaul et al. 2016) on a device sum-tree.
"""
import random as _random


class _Ring:
    """the ring bookkeeping and the reference's sampling, shared by the buffers below (they differ in what a slot stores)"""

    def __init__(self, size, device, rng, seed):
        import torch

        self.torch = torch
        self.size = int(size)
        self.device = torch.device(device)
        self.position = 0
        self.length = 0
        # Modules.py:33 seeds the GLOBAL stream with 20; a caller-supplied generator keeps its own state, seed=None skips seeding
        self.rng = rng if rng is not None else _random
        if rng is None and seed is not None:
            self.rng.seed(seed)

    def __len__(self):
        return self.length

    def _claim(self, n):
        """slots of a push of n transitions in env order -> (skip, idx): the first `skip` transitions are overwritten within the same
        push (n > size) and are not stored; the others go to the slots idx.  Advances the ring."""
        t = self.torch
        skip = max(0, n - self.size)
        if skip:  # only the last `size` survive; the write position still advances by n
            self.position = (self.position + skip) % self.size
            n = self.size
        idx = (self.position + t.arange(n, device=self.device)) % self.size
        self.length = min(self.size, self.length + n)
        self.position = (self.position + n) % self.size
        return skip, idx

    def sample_indices(self, batch_size):
        idx = self.rng.sample(range(self.length), batch_size - 1)
        idx.append((self.position - 1) % self.length)  # memory[position - 1]: the newest (Python's -1 when position == 0)
        return idx


class DeviceReplayBuffer(_Ring):
    def __init__(self, size, state_shape=(4, 200, 200), device="cuda", state_dtype=None, rng=None, seed=20):
        super().__init__(size, device, rng, seed)
        torch = self.torch
        self.states = torch.zeros((self.size,) + tuple(state_shape), dtype=state_dtype or torch.float32, device=self.device)
        self.actions = torch.zeros(self.size, dtype=torch.int64, device=self.device)
        self.rewards = torch.zeros(self.size, dtype=torch.float32, device=self.device)

    def push(self, state, action, reward):
        """one transition: state [4,H,W] or [1,4,H,W] (the agent's tensor), action / reward scalars or 1-element tensors"""
        t = self.torch
        s = state if isinstance(state, t.Tensor) else t.as_tensor(state)
        self.push_batch(s.reshape((1,) + tuple(self.states.shape[1:])), t.as_tensor(action).reshape(1), t.as_tensor(reward).reshape(1))

    def push_batch(self, states, actions, rewards):
        """N transitions in env order = N consecutive `push` calls of the reference (oldest entries are overwritten on wrap-around)"""
        t = self.torch
        n = int(states.shape[0])
        states = states.to(self.device, self.states.dtype)
        actions = t.as_tensor(actions).to(self.device, t.int64).reshape(n)
        rewards = t.as_tensor(rewards).to(self.device, t.float32).reshape(n)
        skip, idx = self._claim(n)
        self.states.index_copy_(0, idx, states[skip:])
        self.actions.index_copy_(0, idx, actions[skip:])
        self.rewards.index_copy_(0, idx, rewards[skip:])

    def sample(self, batch_size):
        """-> (states [B,4,H,W], actions [B,1] int64, rewards [B,1] f32), in the reference's order (random ones, then the newest)"""
        t = self.torch
        idx = t.as_tensor(self.sample_indices(batch_size), dtype=t.int64, device=self.device)
        return self.states.index_select(0, idx), self.actions.index_select(0, idx)[:, None], self.rewards.index_select(0, idx)[:, None]

    def get(self, index):
        return self.states[index], self.actions[index], self.rewards[index]


class ObservationReplay(_Ring):
    """Replay memory of the online trainer: it stores the raw observation (rgb u8 [H,W,3], depth f32 [H,W]), the flat action, the
    reward and the (global env, step) key of each transition - 280 024 B at 200x200 (rgb 120 000, depth 160 000, action int64, reward f32,
    env int64, step int32 holding the uint32 key) against 640 012 B for the f32 state - and
    regenerates the training state at sample time with gq_obs_to_state_keyed.  That transform is a function of the observation and
    its key only, so a sampled state equals, bit for bit, the state the agent acted on when it pushed the transition.  Ring and
    sampling are DeviceReplayBuffer's (the reference's B - 1 uniform picks plus the newest, from `rng`).

    next_obs=True (bootstrapped learning, the reference's `next_state`, Grasping_Agent_multidiscrete.py:140-144,551-554): each
    transition also keeps the observation after its step and that observation's step key (280 004 B more at 200x200: rgb, depth,
    uint32 key; the env is the transition's), and `sample` also returns the regenerated next states.  Off, nothing of it is stored."""

    def __init__(self, size, image_hw=(200, 200), device="cuda", rng=None, seed=20, next_obs=False):
        super().__init__(size, device, rng, seed)
        t = self.torch
        H, W = image_hw
        self.rgb = t.zeros((self.size, H, W, 3), dtype=t.uint8, device=self.device)
        self.depth = t.zeros((self.size, H, W), dtype=t.float32, device=self.device)
        self.actions = t.zeros(self.size, dtype=t.int64, device=self.device)
        self.rewards = t.zeros(self.size, dtype=t.float32, device=self.device)
        self.envs = t.zeros(self.size, dtype=t.int64, device=self.device)
        self.steps = t.zeros(self.size, dtype=t.int32, device=self.device)  # the uint32 step key, bit for bit
        self.next_obs = bool(next_obs)
        self.next_rgb = self.next_depth = self.next_steps = None
        if self.next_obs:
            self.next_rgb = t.zeros_like(self.rgb)
            self.next_depth = t.zeros_like(self.depth)
            self.next_steps = t.zeros_like(self.steps)

    def _key32(self, steps):
        """step keys (any integers) -> the int32 tensor holding their uint32 bit patterns"""
        t = self.torch
        return t.as_tensor(steps).to(t.int64).bitwise_and(0xFFFFFFFF).to(t.int32)

    def push_batch(self, rgb, depth, actions, rewards, envs, steps, next_rgb=None, next_depth=None, next_steps=None):
        """N transitions in env order: observations [N,H,W,3] / [N,H,W], flat actions, rewards, global env ids and the step key; with
        next_obs the observations after the step (next_rgb, next_depth) and their step key (next_steps) too"""
        t = self.torch
        n = int(depth.shape[0])
        if self.next_obs and (next_rgb is None or next_depth is None or next_steps is None):
            raise ValueError("this replay stores next observations: push_batch needs next_rgb, next_depth and next_steps")
        skip, idx = self._claim(n)
        as_dev = lambda x, dt: t.as_tensor(x).to(self.device, dt).reshape(n)[skip:]
        self.rgb.index_copy_(0, idx, rgb[skip:].to(self.device))
        self.depth.index_copy_(0, idx, depth[skip:].to(self.device, t.float32))
        self.actions.index_copy_(0, idx, as_dev(actions, t.int64))
        self.rewards.index_copy_(0, idx, as_dev(rewards, t.float32))
        self.envs.index_copy_(0, idx, as_dev(envs, t.int64))
        self.steps.index_copy_(0, idx, as_dev(self._key32(steps), t.int32))
        if self.next_obs:
            self.next_rgb.index_copy_(0, idx, next_rgb[skip:].to(self.device))
            self.next_depth.index_copy_(0, idx, next_depth[skip:].to(self.device, t.float32))
            self.next_steps.index_copy_(0, idx, as_dev(self._key32(next_steps), t.int32))

    def _states(self, idx, fwd, seed, depth_threshold, noise_std, nxt=False):
        """the keyed training transform of the stored (nxt: next) observations of slots idx"""
        rgb, depth, steps = (self.next_rgb, self.next_depth, self.next_steps) if nxt else (self.rgb, self.depth, self.steps)
        return fwd.obs_to_state_keyed(rgb, depth, self.envs.index_select(0, idx), steps.index_select(0, idx), seed, slot=idx, depth_threshold=depth_threshold,
                                      noise_std=noise_std)

    def sample(self, batch_size, fwd, seed, depth_threshold=1.1, noise_std=0.001):
        """-> (states [B,4,H,W] f32, actions [B,1] int64, rewards [B,1] f32) in the reference's order, with next_obs followed by the
        next states [B,4,H,W] f32; the states are regenerated by `fwd` (a QNetForward on this buffer's device) with the keyed
        transform under `seed`"""
        t = self.torch
        idx = t.as_tensor(self.sample_indices(batch_size), dtype=t.int64, device=self.device)
        out = (self._states(idx, fwd, seed, depth_threshold, noise_std), self.actions.index_select(0, idx)[:, None], self.rewards.index_select(0, idx)[:, None])
        return out + (self._states(idx, fwd, seed, depth_threshold, noise_std, nxt=True),) if self.next_obs else out


class PrioritizedObservationReplay(ObservationReplay):
    """ObservationReplay with proportional prioritized replay (Schaul et al. 2016), on the GPU only (csrc/qnet_replay.cuh).  Slot i is
    drawn with probability p_i / sum p, p_i = (|r - q_pred| + eps)^alpha from the last update that trained on it; a new transition
    enters with the largest priority assigned so far (1.0 at the start).  `tree` [2 cap] f64 is the sum-tree over the slots
    (cap = the smallest power of two >= size) and `pmax` [1] f64 that largest priority; both stay on the device.  The draw is
    stratified (one uniform per 1/B of the total) and keyed on (seed, learner update, rank), so it needs no host generator and no
    host-to-device copy.  Priorities are not part of a checkpoint, like the stored transitions themselves."""

    def __init__(self, size, image_hw=(200, 200), device="cuda", alpha=0.6, eps=1e-6, next_obs=False):
        super().__init__(size, image_hw, device, rng=None, seed=None, next_obs=next_obs)  # the uniform generator is not used (nor the global one re-seeded)
        from .qnet import load_qnet_library
        from .qnet_learn import _bind_learn

        t = self.torch
        if self.device.type != "cuda":
            raise RuntimeError("PrioritizedObservationReplay needs a CUDA device (there is no CPU fallback)")
        self.L = _bind_learn(load_qnet_library())
        self.alpha, self.eps = float(alpha), float(eps)
        self.cap = 1 << max(0, (self.size - 1).bit_length())
        self.tree = t.zeros(2 * self.cap, dtype=t.float64, device=self.device)
        self.pmax = t.ones(1, dtype=t.float64, device=self.device)
        self._claimed = None

    def _ck(self, r, what):
        if r != 0:
            raise RuntimeError(f"{what} failed ({r}): {self.L.gq_last_error().decode()}")

    def _st(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def _claim(self, n):
        skip, idx = super()._claim(n)
        self._claimed = idx
        return skip, idx

    def push_batch(self, rgb, depth, actions, rewards, envs, steps, next_rgb=None, next_depth=None, next_steps=None):
        """ObservationReplay.push_batch, then the claimed slots' priorities := pmax (gq_per_push)"""
        super().push_batch(rgb, depth, actions, rewards, envs, steps, next_rgb, next_depth, next_steps)
        slots = self._claimed.contiguous()
        self._ck(self.L.gq_per_push(self.tree.data_ptr(), self.pmax.data_ptr(), slots.data_ptr(), int(slots.numel()), self.cap, self._st()), "gq_per_push")

    def sample_slots(self, batch_size, beta, seed, update, rank=0):
        """-> (idx [B] int64, importance weights [B] f32), both on the device (gq_per_sample)"""
        t = self.torch
        if self.length == 0:
            raise ValueError("sample from an empty replay")
        idx = t.empty(batch_size, dtype=t.int64, device=self.device)
        w = t.empty(batch_size, dtype=t.float32, device=self.device)
        self._ck(self.L.gq_per_sample(self.tree.data_ptr(), self.cap, self.length, int(batch_size), float(beta), int(seed) & (2 ** 64 - 1),
                                      int(update) & (2 ** 64 - 1), int(rank) & 0xFFFFFFFF, idx.data_ptr(), w.data_ptr(), self._st()), "gq_per_sample")
        return idx, w

    def sample(self, batch_size, fwd, seed, beta, update, rank=0, depth_threshold=1.1, noise_std=0.001):
        """-> (states [B,4,H,W] f32, actions [B,1] int64, rewards [B,1] f32, idx [B] int64, weights [B] f32), with next_obs the next
        states [B,4,H,W] f32 after the rewards; the draw is keyed on (seed, update, rank) - the trainer passes the learner's update
        count and its process rank - and the states are regenerated by `fwd` (a QNetForward on this buffer's device) with the keyed
        transform under `seed`"""
        idx, w = self.sample_slots(batch_size, beta, seed, update, rank)
        out = (self._states(idx, fwd, seed, depth_threshold, noise_std), self.actions.index_select(0, idx)[:, None], self.rewards.index_select(0, idx)[:, None])
        if self.next_obs:
            out += (self._states(idx, fwd, seed, depth_threshold, noise_std, nxt=True),)
        return out + (idx, w)

    def update_priorities(self, idx, qsel, reward):
        """priorities of the slots idx [B] after training on them: (|reward - qsel| + eps)^alpha, in batch order (gq_per_update); `reward`
        is the training target, the Bellman target y when the trainer bootstraps"""
        t = self.torch
        idx = idx.to(self.device, t.int64).reshape(-1).contiguous()
        B = int(idx.numel())
        qsel = qsel.to(self.device, t.float32).reshape(B).contiguous()
        reward = t.as_tensor(reward).to(self.device, t.float32).reshape(B).contiguous()
        self._ck(self.L.gq_per_update(self.tree.data_ptr(), self.pmax.data_ptr(), idx.data_ptr(), qsel.data_ptr(), reward.data_ptr(), B, self.alpha,
                                      self.eps, self.cap, self._st()), "gq_per_update")
