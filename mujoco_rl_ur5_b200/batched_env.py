"""BatchedGraspEnv: N GraspEnv instances stepped together on one GPU.

Host-side mirror of the reference's `GraspEnv` (gym_grasper/envs/GraspingEnv.py:25-489) with a leading env axis:
`reset() -> obs`, `step(action[N,2]) -> (obs, reward[N], done[N], info)`, `render()`.  Action = MultiDiscrete
([W*H, 6]): pixel index and rotation index (GraspingEnv.py:40,94-97,163-165).  Observations stay on the device
(`rgb` u8 [N,H,W,3], `depth` f32 [N,H,W] metres); rewards come back to the host.
"""
import numpy as np

from .engine import BatchedEngine
from .model.scene import load_scene, load_scene_blob

HOME = np.array([0, -1.57, 1.57, -1.57, -1.57, 0.0, 0.3])  # GraspingEnv.py:418
ROTATIONS = {0: 0, 1: 30, 2: 60, 3: 90, 4: -30, 5: -60}   # GraspingEnv.py:40


def scene_a_reset_qpos(arrays, seed):
    """Scene-A reset: the (commented) IT4 rule of GraspingEnv.py:435-463 — every object x~U(-.25,.25), y~U(-.17,.17) around
    the table centre, z = 0, identity orientation; draws in joint order (x then y) from RandomState(seed)."""
    rng = np.random.RandomState(seed)
    q = np.array(arrays["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = HOME[6]
    nobj = (len(q) - 8) // 7
    for i in range(nobj):
        a = 8 + 7 * i
        q[a] = rng.uniform(-0.25, 0.25)
        q[a + 1] = rng.uniform(-0.17, 0.17)
        q[a + 2] = 0.0
        q[a + 3:a + 7] = [1, 0, 0, 0]
    return q


def random_unit_quaternion(r1, r2, r3):
    """pyquaternion's Quaternion.random() from its three uniforms (SURVEY Q8): (w, x, y, z)"""
    s1, s2 = np.sqrt(1.0 - r1), np.sqrt(r1)
    t1, t2 = 2 * np.pi * r2, 2 * np.pi * r3
    return np.array([s1 * np.sin(t1), s1 * np.cos(t1), s2 * np.sin(t2), s2 * np.cos(t2)])


def scene_b_reset_qpos(arrays, seed=None, rng=None):
    """Scene-B reset, the live code of GraspingEnv.py:418-430: 40 free objects, per object x~U(-.25,.25), y~U(-.77,-.43),
    z~U(1.0,1.5), orientation = Quaternion.random() (three more uniforms); draw order x, y, z, r1, r2, r3.  `rng`: a
    RandomState, or numpy's global stream (what the reference uses) when both arguments are None."""
    if rng is None:
        rng = np.random.RandomState(seed) if seed is not None else np.random
    q = np.array(arrays["qpos0"], dtype=np.float64).copy()
    q[:7] = HOME
    q[7] = HOME[6]
    nobj = (len(q) - 8) // 7
    for i in range(nobj):
        a = 8 + 7 * i
        q[a] = rng.uniform(low=-0.25, high=0.25)
        q[a + 1] = rng.uniform(low=-0.77, high=-0.43)
        q[a + 2] = rng.uniform(low=1.0, high=1.5)
        r1, r2, r3 = rng.random_sample(3)
        q[a + 3:a + 7] = random_unit_quaternion(r1, r2, r3)
    return q


class BatchedGraspEnv:
    def __init__(self, n_envs, scene="A", device=0, image_width=200, image_height=200, seed_base=20000, env_index_offset=0,
                 settle_ms=1000):
        import torch

        self.torch = torch
        self.scene = scene
        self.blob = load_scene_blob(scene)
        self.arrays, self.names = load_scene(scene)
        self.engine = BatchedEngine(self.blob, n_envs, device)
        self.n_envs = n_envs
        self.IMAGE_WIDTH, self.IMAGE_HEIGHT = image_width, image_height
        self.TABLE_HEIGHT = 0.91  # GraspingEnv.py:56
        self.rotations = ROTATIONS
        self.cam = int(np.asarray(self.arrays["cam_top_down"]).ravel()[0])
        self.seed_base, self.env_index_offset, self.settle_ms = seed_base, env_index_offset, settle_ms
        self.nvec = np.array([image_width * image_height, len(ROTATIONS)])
        self.current_observation = None
        self.step_called = 0
        self.episode = 0
        self._pin_action = torch.empty((n_envs, 2), dtype=torch.int32).pin_memory()
        self._pin_reward = torch.empty(n_envs, dtype=torch.uint8).pin_memory()
        self._pin_obs = None
        self.h2d_bytes_per_step = self._pin_action.numel() * 4
        self.d2h_bytes_per_step = self._pin_reward.numel()
        self.obs_bytes = n_envs * image_width * image_height * (3 + 4)  # rgb u8 x3 + depth f32
        self._branch = None  # engine of evaluate_actions, created at its first call

    # ------------------------------------------------------------------ gym-like API
    def reset(self):
        """GraspEnv.reset_model (GraspingEnv.py:409-477): randomise objects, arm to HOME, settle, observe."""
        seeds = self.seed_base + self.env_index_offset + np.arange(self.n_envs) + 100003 * self.episode
        rule = scene_b_reset_qpos if self.scene == "B" else scene_a_reset_qpos
        q = np.stack([rule(self.arrays, int(s)) for s in seeds])
        self.episode += 1
        eng = self.engine
        eng.set_state(q)
        eng.stay(self.settle_ms)
        eng.run()
        # unlike the reference (quirk Q5: GraspEnv.reset leaves current_observation stale) the batched API acts on what it returns
        self.current_observation = self.get_observation()
        return self.current_observation

    def get_observation(self):
        rgb, depth = self.engine.render(self.cam, self.IMAGE_WIDTH, self.IMAGE_HEIGHT)
        return {"rgb": rgb, "depth": depth}

    def step(self, action, obs_to_host=False):
        """action: int array [N,2] (host).  Returns (obs, reward u8[N] host, done bool[N], info).  obs_to_host=True additionally
        copies the new observation into pinned host buffers (`info["obs_host"]`), which is what the reference's single-env API hands
        its caller every step; by default observations stay on the device for a device-side agent."""
        t = self.torch
        eng = self.engine
        if self.current_observation is None or self.step_called == 1:
            self.current_observation = self.get_observation()  # GraspingEnv.py:87-88
        if isinstance(action, t.Tensor) and action.is_cuda:  # actions already on the device (e.g. from BatchedGreedyAgent)
            act = action.to(t.int32).reshape(self.n_envs, 2)
        else:
            self._pin_action.copy_(t.as_tensor(np.asarray(action, dtype=np.int32).reshape(self.n_envs, 2)))
            act = self._pin_action.to(eng.device, non_blocking=True)
        W = self.IMAGE_WIDTH
        x = act[:, 0] % W
        y = t.div(act[:, 0], W, rounding_mode="floor")
        rot = act[:, 1].contiguous()
        depth = self.current_observation["depth"]
        d = depth[t.arange(self.n_envs, device=eng.device), y.long(), x.long()].contiguous()
        coords = eng.pixel_2_world(x.contiguous(), y.contiguous(), d, self.cam, W, self.IMAGE_HEIGHT)
        # "Skipping execution due to bad depth value!" (GraspingEnv.py:124-131)
        execute = ~((coords[:, 2] < 0.8) | (coords[:, 1] > -0.3))
        eng.grasp(coords, rot, self.TABLE_HEIGHT, env_mask=execute.to(t.uint8))
        eng.run()
        _, _, reward, _ = eng.results()
        reward = reward * execute.to(t.uint8)
        self._pin_reward.copy_(reward, non_blocking=True)
        self.current_observation = self.get_observation()
        info = {"executed": execute}
        if obs_to_host:
            if self._pin_obs is None:
                self._pin_obs = {k: t.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in self.current_observation.items()}
            for k, v in self.current_observation.items():
                self._pin_obs[k].copy_(v, non_blocking=True)
            info["obs_host"] = self._pin_obs
        t.cuda.current_stream().synchronize()
        self.step_called += 1
        return self.current_observation, self._pin_reward.numpy().copy(), np.zeros(self.n_envs, bool), info

    # ------------------------------------------------------------------ whole states (env_state.py)
    def snapshot(self):
        """EngineState of every env plus what this façade keeps beside the engine (current observation, step counter, episode), so
        that a restored env's next `step` is the original's next `step`"""
        s = self.engine.snapshot()
        obs = None if self.current_observation is None else {k: v.clone() for k, v in self.current_observation.items()}
        s.facade = {"observation": obs, "step_called": self.step_called, "episode": self.episode}
        return s

    def restore(self, s):
        """puts back a `snapshot` (also one loaded with EngineState.load); raises EngineError, leaving everything as it was, for a
        snapshot of another scene"""
        self.engine.restore(s)
        if s.facade is not None:
            obs = s.facade.get("observation")
            self.current_observation = None if obs is None else {k: v.to(self.engine.device).clone() for k, v in obs.items()}
            self.step_called, self.episode = int(s.facade["step_called"]), int(s.facade["episode"])

    def evaluate_actions(self, actions, max_branch_envs=4096):
        """Grasp outcome of K candidate actions per env from the env's current state, without changing it: actions [N, K, 2] (pixel
        index, rotation index as `step` takes them) -> (reward u8 [N, K], executed bool [N, K]) on the device.  Pixels turn into
        world points as in `step` (the current observation's depth, bad-depth attempts skipped with reward 0); the N*K attempts run in
        a second engine of the same scene, restored from this one's snapshot, at most `max_branch_envs` at a time.  Attempt (e, k) is
        bit for bit what `step` would give with action k."""
        t = self.torch
        eng = self.engine
        act = t.as_tensor(actions).to(device=eng.device, dtype=t.int32)
        N, K = act.shape[0], act.shape[1]
        if act.shape != (self.n_envs, K, 2) or K < 1 or max_branch_envs < 1:
            raise ValueError(f"actions must be [{self.n_envs}, K, 2] and max_branch_envs >= 1, got {tuple(act.shape)}, {max_branch_envs}")
        obs = self.current_observation if self.current_observation is not None else self.get_observation()
        W, H = self.IMAGE_WIDTH, self.IMAGE_HEIGHT
        ar = t.arange(N, device=eng.device)
        coords = t.empty((N, K, 3), dtype=t.float64, device=eng.device)
        for k in range(K):
            x = act[:, k, 0] % W
            y = t.div(act[:, k, 0], W, rounding_mode="floor")
            d = obs["depth"][ar, y.long(), x.long()].contiguous()
            coords[:, k] = eng.pixel_2_world(x.contiguous(), y.contiguous(), d, self.cam, W, H)
        execute = ~((coords[..., 2] < 0.8) | (coords[..., 1] > -0.3))  # as in step
        coords, rot, execute = coords.reshape(N * K, 3), act[..., 1].reshape(N * K), execute.reshape(N * K)
        B = min(N * K, int(max_branch_envs))
        if self._branch is None or self._branch.n_envs != B:
            if self._branch is not None:
                self._branch.close()
            self._branch = BatchedEngine(self.blob, B, eng.device.index or 0)
        br = self._branch
        state = eng.snapshot()
        reward = t.zeros(N * K, dtype=t.uint8, device=eng.device)
        slot = t.arange(B, device=eng.device)
        for j0 in range(0, N * K, B):
            n = min(B, N * K - j0)
            live = slot < n
            rows = t.where(live, t.div(j0 + slot, K, rounding_mode="floor"), t.full_like(slot, -1))
            br.restore(state, rows)
            pad = lambda a: t.cat([a[j0:j0 + n], a[:B - n]]) if n < B else a[j0:j0 + n]
            mask = pad(execute) & live
            br.grasp(pad(coords).contiguous(), pad(rot).contiguous(), self.TABLE_HEIGHT, env_mask=mask.to(t.uint8))
            br.run()
            reward[j0:j0 + n] = (br.results()[2] * mask.to(t.uint8))[:n]
        return reward.reshape(N, K), execute.reshape(N, K)

    def render(self, mode="rgb_array"):
        return self.get_observation()["rgb"]

    def sample_actions(self, rng):
        return np.stack([rng.randint(0, self.nvec[0], self.n_envs), rng.randint(0, self.nvec[1], self.n_envs)], axis=1)

    def total_substeps(self):
        return int(self.engine.results()[3].sum().item())

    def close(self):
        self.engine.close()
        if self._branch is not None:
            self._branch.close()
