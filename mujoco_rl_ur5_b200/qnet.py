"""Pixel-wise grasp Q-network: weights container + batched bf16 forward on the in-tree CUDA library (libgrasp_qnet.so).

Reference: Modules.py:308-311 `MULTIDISCRETE_RESNET(number_actions_dim_2)` = nn.Sequential(Perception_Module (:159-193),
Grasping_Module_multidiscrete (:243-287)), built from BasicBlock (:92-142) and conv3x3 (:145-156).

* `make_torch_qnet()` re-declares the architecture with the reference's attribute names and construction order, so that
  (a) `torch.manual_seed(s)` gives bit-identical initial weights to the reference module and (b) the reference's checkpoints
  (`model_state_dict`, Grasping_Agent_multidiscrete.py:560-572) load with `load_state_dict`.  It is a weights container and the
  fp32 comparison target of the tests — the product forward never calls it.
* `QNetForward` packs the weights once (bf16, [Cout][kh][kw][Cin]) and runs the whole forward with the hand-written kernels:
  wgmma implicit-GEMM convolutions + fused BN/ReLU/residual, max-pool, bilinear up-sampling, sigmoid head, arg-max.
  BatchNorm uses per-image batch statistics: the reference never calls `.eval()` on the policy net and forwards one image at a
  time (SURVEY 3.4, Q9), so a batch of N environments is N independent batch-1 forwards.
* `QNetForward(..., batchnorm="running")` is the eval-mode forward (`policy_net.eval()`, Offline RL/train.py:172): BatchNorm with the
  running statistics is a per-channel affine map, folded into the convolution weights when they are packed, so a BasicBlock is two
  wgmma launches (gq_conv_tc_fused) with bf16 outputs and no fp32 intermediates.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
QLIB_PATH = os.path.join(_HERE, "csrc", "libgrasp_qnet.so")
_QLIB = None
QSYMBOLS = ["gq_last_error", "gq_version", "gq_conv_partials_floats", "gq_conv_tc", "gq_conv_tc_block_out", "gq_conv_first", "gq_maxpool", "gq_bn_act", "gq_upsample2x", "gq_head_up2", "gq_argmax", "gq_obs_to_state", "gq_obs_to_state_train", "gq_conv_tc_fused",
            "gq_obs_to_state_keyed", "gq_sample_actions", "gq_head_max_target", "gq_obs_to_state_standard", "gq_obs_channel_stats",
            "gq_obs_channel_stats_scratch_bytes"]


def load_qnet_library():
    global _QLIB
    if _QLIB is None:
        if not os.path.exists(QLIB_PATH):
            raise RuntimeError(f"{QLIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(QLIB_PATH)
        P, I, F = C.c_void_p, C.c_int, C.c_float
        L.gq_last_error.restype = C.c_char_p
        L.gq_version.restype = C.c_char_p
        L.gq_conv_partials_floats.argtypes = [I, I, I, I]
        L.gq_conv_partials_floats.restype = C.c_size_t
        L.gq_conv_tc.argtypes = [P, P, P, P, P, P, I, I, I, I, I, I, P]
        L.gq_conv_tc_block_out.argtypes = [P, P, P, P, P, P, P, F, P, P, I, I, I, I, I, I, P]
        L.gq_conv_tc_fused.argtypes = [P, P, P, P, P, I, I, I, I, I, I, I, I, P]
        L.gq_conv_first.argtypes = [P, P, P, I, I, I, P]
        L.gq_maxpool.argtypes = [P, P, I, I, I, I, P]
        L.gq_bn_act.argtypes = [P, P, P, P, P, P, I, I, I, F, P]
        L.gq_upsample2x.argtypes = [P, P, I, I, I, I, P]
        L.gq_head_up2.argtypes = [P, P, P, P, P, I, I, I, I, P]
        L.gq_argmax.argtypes = [P, I, I, P, P, P]
        L.gq_head_max_target.argtypes = [P, P, P, P, F, P, P, I, I, I, I, P]
        L.gq_obs_to_state.argtypes = [P, P, F, P, P, I, I, P]
        L.gq_obs_to_state_train.argtypes = [P, P, F, F, C.c_uint64, P, C.c_uint32, P, P, P, P, P, I, I, P]
        L.gq_obs_to_state_keyed.argtypes = [P, P, P, P, P, F, F, C.c_uint64, P, P, P, P, P, I, I, P]
        L.gq_obs_to_state_standard.argtypes = [P, P, P, P, P, C.c_uint32, P, F, F, C.c_uint64, P, P, I, I, P]
        L.gq_obs_channel_stats_scratch_bytes.argtypes = [C.c_longlong]
        L.gq_obs_channel_stats_scratch_bytes.restype = C.c_size_t
        L.gq_obs_channel_stats.argtypes = [P, P, I, I, P, P, P]
        D = C.c_double
        L.gq_sample_actions.argtypes = [P, P, P, C.c_uint64, P, C.c_uint32, D, P, P, D, I, I, I, I, I, P, P, P, P]
        _QLIB = L
    return _QLIB


def make_torch_qnet(number_actions_dim_2=6):
    """torch.nn re-declaration of MULTIDISCRETE_RESNET with the reference's parameter names and creation order."""
    import torch.nn as nn

    def conv3x3(i, o):
        return nn.Conv2d(i, o, kernel_size=3, stride=1, padding=1, bias=False)

    class BasicBlock(nn.Module):
        def __init__(self, inplanes, planes):
            super().__init__()
            self.conv1 = conv3x3(inplanes, planes)
            self.bn1 = nn.BatchNorm2d(planes)
            self.relu = nn.ReLU(inplace=True)
            self.conv2 = conv3x3(planes, planes)
            self.bn2 = nn.BatchNorm2d(planes)
            self.conv3 = nn.Conv2d(inplanes, planes, kernel_size=1, stride=1) if inplanes != planes else None

        def forward(self, x):
            identity = x
            out = self.relu(self.bn1(self.conv1(x)))
            out = self.bn2(self.conv2(out))
            if self.conv3 is not None:
                identity = self.conv3(identity)
            return self.relu(out + identity)

    class Perception_Module(nn.Module):
        def __init__(self):
            super().__init__()
            self.C1 = conv3x3(4, 64)
            self.MP1 = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
            self.RB1 = BasicBlock(64, 128)
            self.MP2 = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
            self.RB2 = BasicBlock(128, 256)
            self.RB3 = BasicBlock(256, 512)

        def forward(self, x):
            return self.RB3(self.RB2(self.MP2(self.RB1(self.MP1(self.C1(x))))))

    class Grasping_Module_multidiscrete(nn.Module):
        def __init__(self, act_dim_2):
            super().__init__()
            self.RB1 = BasicBlock(512, 256)
            self.RB2 = BasicBlock(256, 128)
            self.UP1 = nn.UpsamplingBilinear2d(scale_factor=2)
            self.RB3 = BasicBlock(128, 64)
            self.UP2 = nn.UpsamplingBilinear2d(scale_factor=2)
            self.C1 = nn.Conv2d(64, act_dim_2, kernel_size=1)
            self.sigmoid = nn.Sigmoid()

        def forward(self, x):
            x = self.C1(self.UP2(self.RB3(self.UP1(self.RB2(self.RB1(x))))))
            return self.sigmoid(x.squeeze())

    return nn.Sequential(Perception_Module(), Grasping_Module_multidiscrete(number_actions_dim_2))


_BLOCKS = ["0.RB1", "0.RB2", "0.RB3", "1.RB1", "1.RB2", "1.RB3"]
BN_EPS = 1e-5


def fold_block_weights(sd, name, eps=BN_EPS):
    """eval-mode BasicBlock `name` with BatchNorm folded into the convolutions, in fp32 (s = gamma * rsqrt(running_var + eps)):
    -> (w1 [Cout,Cin,3,3] = W1 s1, bias1 [Cout] = beta1 - mu1 s1, w2 [Cout,Cout,3,3] = W2 s2, bias2 [Cout] = beta2 - mu2 s2 + b3)"""
    s1 = sd[f"{name}.bn1.weight"] * (sd[f"{name}.bn1.running_var"] + eps).rsqrt()
    s2 = sd[f"{name}.bn2.weight"] * (sd[f"{name}.bn2.running_var"] + eps).rsqrt()
    w1 = sd[f"{name}.conv1.weight"] * s1[:, None, None, None]
    w2 = sd[f"{name}.conv2.weight"] * s2[:, None, None, None]
    b1 = sd[f"{name}.bn1.bias"] - sd[f"{name}.bn1.running_mean"] * s1
    b2 = sd[f"{name}.bn2.bias"] - sd[f"{name}.bn2.running_mean"] * s2 + sd[f"{name}.conv3.bias"]
    return w1, b1, w2, b2


class QNetForward:
    """Batched forward on cuda.  `state_dict` uses the reference's key names ('0.C1.weight', '0.RB1.conv1.weight', ...).

    batchnorm="batch" (default): training-mode BatchNorm with each image's own statistics, what the reference's acting forward computes.
    batchnorm="running": eval-mode BatchNorm with the state_dict's running_mean / running_var (ValueError if it has none), folded into
    the convolution weights; then the Q-map of an image does not depend on the other images of the batch or on `max_batch`."""

    def __init__(self, state_dict, device=0, max_batch=64, batchnorm="batch"):
        import torch

        if batchnorm not in ("batch", "running"):
            raise ValueError(f"batchnorm must be 'batch' or 'running', not {batchnorm!r}")
        if batchnorm == "running":
            missing = [f"{n}.{bn}.{s}" for n in _BLOCKS for bn in ("bn1", "bn2") for s in ("running_mean", "running_var") if f"{n}.{bn}.{s}" not in state_dict]
            if missing:
                raise ValueError(f"batchnorm='running' needs the BatchNorm running statistics; the state_dict has no {missing[0]} (and {len(missing) - 1} more)")
        if not torch.cuda.is_available():
            raise RuntimeError("QNetForward needs a CUDA device (there is no CPU fallback)")
        self.torch = torch
        self.L = load_qnet_library()
        self.dev = torch.device("cuda", device)
        self.max_batch = max_batch
        self.batchnorm = batchnorm
        sd = {k: v.detach().to(self.dev, torch.float32) for k, v in state_dict.items()}
        self.A = sd["1.C1.weight"].shape[0]
        pack = lambda w: w.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)  # [Cout,Cin,kh,kw] -> [Cout,kh,kw,Cin]
        self.w_first = sd["0.C1.weight"].permute(0, 2, 3, 1).contiguous()       # [64,3,3,4] f32
        self.blocks = []
        for name in _BLOCKS:
            cin, cout = sd[f"{name}.conv1.weight"].shape[1], sd[f"{name}.conv1.weight"].shape[0]
            if batchnorm == "running":
                # folded in fp32, rounded to bf16 once; launch 2's weights are [W2 s2 | W3] = one [Cout][9 Cout + Cin] matrix
                w1, b1, w2, b2 = fold_block_weights(sd, name)
                w23 = torch.cat([w2.permute(0, 2, 3, 1).reshape(cout, 9 * cout), sd[f"{name}.conv3.weight"].reshape(cout, cin)], dim=1)
                b = dict(fw1=pack(w1), fb1=b1.contiguous(), fw23=w23.contiguous().to(torch.bfloat16), fb2=b2.contiguous(), cin=cin, cout=cout)
            else:
                b = dict(w1=pack(sd[f"{name}.conv1.weight"]), w2=pack(sd[f"{name}.conv2.weight"]), w3=pack(sd[f"{name}.conv3.weight"]),
                         b3=sd[f"{name}.conv3.bias"].contiguous(), g1=sd[f"{name}.bn1.weight"].contiguous(), be1=sd[f"{name}.bn1.bias"].contiguous(),
                         g2=sd[f"{name}.bn2.weight"].contiguous(), be2=sd[f"{name}.bn2.bias"].contiguous(), cin=cin, cout=cout)
            self.blocks.append(b)
        self.w_head = sd["1.C1.weight"].reshape(self.A, 64).contiguous()
        self.b_head = sd["1.C1.bias"].contiguous()
        self.launches = 0

    def _ck(self, r, what):
        if r != 0:
            raise RuntimeError(f"{what} failed ({r}): {self.L.gq_last_error().decode()}")
        self.launches += 1

    def _p(self, t):
        return None if t is None else C.c_void_p(t.data_ptr())

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.dev).cuda_stream)

    # ---- layer wrappers (also used one by one by the parity tests)
    def conv_tc(self, x, w, bias, B, H, W, cin, cout, ks, want_stats):
        t = self.torch
        y = t.empty((B, H, W, cout), dtype=t.float32, device=self.dev)
        stats = t.empty((B, cout, 2), dtype=t.float32, device=self.dev) if want_stats else None
        part = t.empty(self.L.gq_conv_partials_floats(B, H, W, cout), dtype=t.float32, device=self.dev) if want_stats else None
        self._ck(self.L.gq_conv_tc(self._p(x), self._p(w), self._p(bias), self._p(y), self._p(stats), self._p(part), B, H, W, cin, cout, ks, self._stream()), "gq_conv_tc")
        return y, stats

    def conv_tc_block_out(self, x, w, bias, resid, stats, gamma, beta, B, H, W, cin, cout, ks=1):
        """relu(BN(resid; per-image stats, gamma, beta) + conv(x, w) + bias) -> bf16 [B, H*W, cout]: the tail of BasicBlock.forward
        (Modules.py:136-142) with the shortcut convolution's epilogue doing the normalisation, the add and the ReLU"""
        t = self.torch
        y = t.empty((B, H * W, cout), dtype=t.bfloat16, device=self.dev)
        ss = t.empty((B, cout, 2), dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_conv_tc_block_out(self._p(x), self._p(w), self._p(bias), self._p(resid), self._p(stats), self._p(gamma), self._p(beta), 1e-5,
                                              self._p(ss), self._p(y), B, H, W, cin, cout, ks, self._stream()), "gq_conv_tc_block_out")
        return y

    def bn_act(self, x, stats, gamma, beta, identity, B, HW, Cc):
        t = self.torch
        y = t.empty((B, HW, Cc), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_bn_act(self._p(x), self._p(stats), self._p(gamma), self._p(beta), self._p(identity), self._p(y), B, HW, Cc, 1e-5, self._stream()), "gq_bn_act")
        return y

    def conv_tc_fused(self, a, x, w, bias, B, H, W, ca, cx, cout, ks=3, relu=True):
        """[relu](conv_ks(a) + conv1x1(x) + bias) -> bf16 [B, H*W, cout] in one wgmma launch; w [cout][ks*ks*ca + cx] bf16, x None when cx = 0"""
        t = self.torch
        y = t.empty((B, H * W, cout), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_conv_tc_fused(self._p(a), self._p(x), self._p(w), self._p(bias), self._p(y), int(relu), B, H, W, ca, cx, cout, ks, self._stream()),
                 "gq_conv_tc_fused")
        return y

    def basic_block(self, x, blk, B, H, W):
        """BasicBlock.forward (Modules.py:128-142) on NHWC bf16 `x`"""
        cin, cout = blk["cin"], blk["cout"]
        if self.batchnorm == "running":
            a1 = self.conv_tc_fused(x, None, blk["fw1"], blk["fb1"], B, H, W, cin, 0, cout)
            return self.conv_tc_fused(a1, x, blk["fw23"], blk["fb2"], B, H, W, cout, cin, cout)
        o1, s1 = self.conv_tc(x, blk["w1"], None, B, H, W, cin, cout, 3, True)
        a1 = self.bn_act(o1, s1, blk["g1"], blk["be1"], None, B, H * W, cout)
        o2, s2 = self.conv_tc(a1, blk["w2"], None, B, H, W, cout, cout, 3, True)
        return self.conv_tc_block_out(x, blk["w3"], blk["b3"], o2, s2, blk["g2"], blk["be2"], B, H, W, cin, cout, 1)

    def maxpool(self, x, B, H, W, Cc):
        t = self.torch
        y = t.empty((B, (H + 1) // 2, (W + 1) // 2, Cc), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_maxpool(self._p(x), self._p(y), B, H, W, Cc, self._stream()), "gq_maxpool")
        return y

    def upsample(self, x, B, H, W, Cc):
        t = self.torch
        y = t.empty((B, 2 * H, 2 * W, Cc), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_upsample2x(self._p(x), self._p(y), B, H, W, Cc, self._stream()), "gq_upsample2x")
        return y

    def _trunk(self, state):
        """every layer up to the head: state [B,4,H,W] f32 -> (x [B,H/2,W/2,64] bf16, the input of UP2 and C1, its height, its width)"""
        t = self.torch
        B, _, H, W = state.shape
        x = t.empty((B, H, W, 64), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_conv_first(self._p(state), self._p(self.w_first), self._p(x), B, H, W, self._stream()), "gq_conv_first")
        x = self.maxpool(x, B, H, W, 64)
        h, w = (H + 1) // 2, (W + 1) // 2
        x = self.basic_block(x, self.blocks[0], B, h, w)            # 0.RB1 64->128 @100
        x = self.maxpool(x, B, h, w, 128)
        h2, w2 = (h + 1) // 2, (w + 1) // 2
        x = self.basic_block(x, self.blocks[1], B, h2, w2)          # 0.RB2 128->256 @50
        x = self.basic_block(x, self.blocks[2], B, h2, w2)          # 0.RB3 256->512
        x = self.basic_block(x, self.blocks[3], B, h2, w2)          # 1.RB1 512->256
        x = self.basic_block(x, self.blocks[4], B, h2, w2)          # 1.RB2 256->128
        x = self.upsample(x.view(B, h2, w2, 128), B, h2, w2, 128)   # -> 100
        x = self.basic_block(x, self.blocks[5], B, 2 * h2, 2 * w2)  # 1.RB3 128->64
        return x, 2 * h2, 2 * w2

    def _head(self, x, h, w):
        """UP2 -> C1 -> sigmoid on the head input x [B,h,w,64] bf16 -> Q [B,A,2h,2w] f32"""
        t = self.torch
        B = x.shape[0]
        q = t.empty((B, self.A, 2 * h, 2 * w), dtype=t.float32, device=self.dev)
        z = t.empty((B, self.A, h, w), dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_head_up2(self._p(x), self._p(self.w_head), self._p(self.b_head), self._p(z), self._p(q), B, h, w, self.A, self._stream()),
                 "gq_head_up2")
        return q

    def _forward_chunk(self, state):
        return self._head(*self._trunk(state))

    def forward(self, state):
        """state [B,4,H,W] f32 on the device -> Q [B,A,H,W] f32 (sigmoid), chunked to bound activation memory"""
        t = self.torch
        state = state.to(self.dev, t.float32).contiguous()
        outs = [self._forward_chunk(state[i:i + self.max_batch]) for i in range(0, state.shape[0], self.max_batch)]
        return outs[0] if len(outs) == 1 else t.cat(outs, dim=0)

    def max_target(self, state, reward, gamma):
        """the bootstrapped target of learn() (Grasping_Agent_multidiscrete.py:430-437) with this network as the target network:
        state [B,4,H,W] f32 (the next states), reward [B] -> (qmax [B] f32 = Q(state).view(B, -1).max(1)[0], y [B] f32 =
        min(1, reward + gamma * qmax) with gamma rounded to f32 and the product and the sum rounded separately).  Chunked like
        `forward`; the Q-maps are never written (gq_head_max_target)."""
        t = self.torch
        state = state.to(self.dev, t.float32).contiguous()
        B = state.shape[0]
        reward = t.as_tensor(reward).to(self.dev, t.float32).reshape(B).contiguous()
        qmax = t.empty(B, dtype=t.float32, device=self.dev)
        y = t.empty(B, dtype=t.float32, device=self.dev)
        for i in range(0, B, self.max_batch):
            x, h, w = self._trunk(state[i:i + self.max_batch])
            self._ck(self.L.gq_head_max_target(self._p(x), self._p(self.w_head), self._p(self.b_head), self._p(reward[i:]), float(gamma), self._p(qmax[i:]),
                                               self._p(y[i:]), x.shape[0], h, w, self.A, self._stream()), "gq_head_max_target")
        return qmax, y

    def obs_to_state(self, obs, depth_threshold=1.1):
        """batched deterministic transform_observation: obs dict of device tensors (rgb u8 [B,H,W,3], depth f32 [B,H,W]) -> [B,4,H,W] f32.
        depth_threshold = cam height - TABLE_HEIGHT + 0.01 = 1.1 (Grasping_Agent_multidiscrete.py:130-135)"""
        t = self.torch
        rgb, depth = obs["rgb"].contiguous(), obs["depth"].contiguous()
        B, H, W = depth.shape
        state = t.empty((B, 4, H, W), dtype=t.float32, device=self.dev)
        mm = t.empty((B, 2), dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_obs_to_state(self._p(rgb), self._p(depth), float(depth_threshold), self._p(mm), self._p(state), B, H * W, self._stream()), "gq_obs_to_state")
        self.launches += 1
        return state

    def draw_color_jitter(self, B, generator=None, brightness=0.5, contrast=0.5, saturation=0.5, hue=0.5):
        """per-image ColorJitter parameters exactly as torchvision's ColorJitter.get_params draws them (randperm(4), then the four
        uniforms, per image; Grasping_Agent_multidiscrete.py:121): -> (factors [B,4] f32, order [B,4] int32) on the device"""
        t = self.torch
        fac, order = [], []
        for _ in range(B):
            order.append(t.randperm(4, generator=generator))
            fac.append(t.stack([t.empty(1).uniform_(1 - brightness, 1 + brightness, generator=generator)[0],
                                t.empty(1).uniform_(1 - contrast, 1 + contrast, generator=generator)[0],
                                t.empty(1).uniform_(1 - saturation, 1 + saturation, generator=generator)[0],
                                t.empty(1).uniform_(-hue, hue, generator=generator)[0]]))
        return t.stack(fac).to(self.dev, t.float32).contiguous(), t.stack(order).to(self.dev, t.int32).contiguous()

    def obs_to_state_train(self, obs, depth_threshold=1.1, noise_std=0.001, seed=0, step=0, env_index=None, jitter=None, order=None, nhwc_bf16=False):
        """transform_observation as the LEARNING agent calls it (normalize=True, jitter_and_noise=True), batched on the device: depth noise
        N(0, noise_std) from a counter-based generator keyed on (seed, global env id, step, pixel) added before the min-max normalisation,
        ColorJitter with the given per-image factors / operation order (see draw_color_jitter; None = no colour change).
        -> [B,4,H,W] f32, or ([B,4,H,W] f32, [B,H,W,4] bf16 NHWC) with nhwc_bf16=True"""
        t = self.torch
        rgb, depth = obs["rgb"].contiguous(), obs["depth"].contiguous()
        B, H, W = depth.shape
        state = t.empty((B, 4, H, W), dtype=t.float32, device=self.dev)
        nhwc = t.empty((B, H, W, 4), dtype=t.bfloat16, device=self.dev) if nhwc_bf16 else None
        red = t.empty((B, 4), dtype=t.float32, device=self.dev)
        ei = None if env_index is None else t.as_tensor(env_index).to(self.dev, t.int64).contiguous()
        self._ck(self.L.gq_obs_to_state_train(self._p(rgb), self._p(depth), float(depth_threshold), float(noise_std), int(seed) & (2 ** 64 - 1), self._p(ei),
                                              int(step) & 0xFFFFFFFF, self._p(jitter), self._p(order), self._p(red), self._p(state), self._p(nhwc), B, H * W,
                                              self._stream()), "gq_obs_to_state_train")
        self.launches += 1
        return (state, nhwc) if nhwc_bf16 else state

    def obs_to_state_keyed(self, rgb, depth, env_index, step, seed, slot=None, depth_threshold=1.1, noise_std=0.001, return_draws=False):
        """the training transform with the ColorJitter factors and order drawn from the keyed generator (gq_obs_to_state_keyed): row b is
        image slot[b] of rgb [S,H,W,3] u8 / depth [S,H,W] f32 (slot None: b), keyed on env_index[b] and step[b] (int64 / uint32 tensors
        or sequences of B).  -> state [B,4,H,W] f32, and (factors [B,4] f32, order [B,4] int32) with return_draws=True"""
        t = self.torch
        rgb, depth = rgb.contiguous(), depth.contiguous()
        H, W = depth.shape[1], depth.shape[2]
        ei = t.as_tensor(env_index).to(self.dev, t.int64).contiguous()
        B = ei.numel()
        st = t.as_tensor(step).to(self.dev, t.int64).reshape(B).bitwise_and(0xFFFFFFFF).to(t.int32).contiguous()  # the uint32 bit pattern
        sl = None if slot is None else t.as_tensor(slot).to(self.dev, t.int64).contiguous()
        state = t.empty((B, 4, H, W), dtype=t.float32, device=self.dev)
        red = t.empty((B, 4), dtype=t.float32, device=self.dev)
        fac = t.empty((B, 4), dtype=t.float32, device=self.dev)
        order = t.empty((B, 4), dtype=t.int32, device=self.dev)
        self._ck(self.L.gq_obs_to_state_keyed(self._p(rgb), self._p(depth), self._p(sl), self._p(ei), self._p(st), float(depth_threshold), float(noise_std),
                                              int(seed) & (2 ** 64 - 1), self._p(red), self._p(fac), self._p(order), self._p(state), None, B, H * W,
                                              self._stream()), "gq_obs_to_state_keyed")
        return (state, fac, order) if return_draws else state

    def obs_to_state_standard(self, obs, stats, depth_threshold=1.1, noise_std=0.001, seed=0, step=0, env_index=None, nhwc_bf16=False, slot=None):
        """transform_observation(normalize=False) batched (gq_obs_to_state_standard): each channel standardised with `stats`, the 8 values
        of normalize.py (obs_stats; mean r, g, b, depth, std r, g, b, depth, rounded to f32 as torchvision's Normalize does), rgb in
        0..255, depth clipped at depth_threshold, then + noise_std * N(0, 1) keyed on (seed, env, step, pixel) as the training transform's
        noise.  No ColorJitter.  Row b is image slot[b] of obs (None: b), keyed on env_index[b] (None: b) and step (an int, or [B] per
        row).  noise_std=0 gives the deterministic part.  -> [B,4,H,W] f32, or ([B,4,H,W] f32, [B,H,W,4] bf16 NHWC) with nhwc_bf16=True"""
        from .obs_stats import as_float32

        t = self.torch
        ms = as_float32(stats)
        rgb, depth = obs["rgb"].contiguous(), obs["depth"].contiguous()
        H, W = depth.shape[1], depth.shape[2]
        sl = None if slot is None else t.as_tensor(slot).to(self.dev, t.int64).reshape(-1).contiguous()
        B = depth.shape[0] if sl is None else sl.numel()
        ei = None if env_index is None else t.as_tensor(env_index).to(self.dev, t.int64).reshape(B).contiguous()
        st = None
        if isinstance(step, (int, np.integer)):
            step = int(step) & 0xFFFFFFFF
        else:  # per row: the uint32 bit patterns
            st = t.as_tensor(step).to(self.dev, t.int64).reshape(B).bitwise_and(0xFFFFFFFF).to(t.int32).contiguous()
            step = 0
        state = t.empty((B, 4, H, W), dtype=t.float32, device=self.dev)
        nhwc = t.empty((B, H, W, 4), dtype=t.bfloat16, device=self.dev) if nhwc_bf16 else None
        self._ck(self.L.gq_obs_to_state_standard(self._p(rgb), self._p(depth), self._p(sl), self._p(ei), self._p(st), step,
                                                 ms.ctypes.data_as(C.c_void_p), float(depth_threshold), float(noise_std), int(seed) & (2 ** 64 - 1),
                                                 self._p(state), self._p(nhwc), B, H * W, self._stream()), "gq_obs_to_state_standard")
        return (state, nhwc) if nhwc_bf16 else state

    def sample_actions(self, depth, greedy_idx, eps, env_index, step, seed, camera, z_min, n_rot=6, max_draws=256):
        """epsilon-greedy selection (gq_sample_actions): depth [B,H,W] f32 of the current observation, greedy_idx [B] int32 (flat arg-max),
        eps [B] f64, env_index [B] int64 global env ids, step / seed: the keyed generator's counter and key, camera = (fovy, pos[3],
        mat[9]) of the top-down camera, z_min = TABLE_HEIGHT - 0.01.  -> (action [B,2] int32, is_random [B] bool, exhausted [B] bool)"""
        t = self.torch
        B, H, W = depth.shape
        depth = depth.contiguous()
        gi = greedy_idx.to(self.dev, t.int32).contiguous()
        ep = t.as_tensor(eps, dtype=t.float64).to(self.dev).reshape(B).contiguous()
        ei = t.as_tensor(env_index).to(self.dev, t.int64).reshape(B).contiguous()
        fovy, pos, mat = camera
        pos = (C.c_double * 3)(*[float(v) for v in np.asarray(pos).ravel()])
        mat = (C.c_double * 9)(*[float(v) for v in np.asarray(mat).ravel()])
        action = t.empty((B, 2), dtype=t.int32, device=self.dev)
        rnd = t.empty(B, dtype=t.uint8, device=self.dev)
        exh = t.empty(B, dtype=t.uint8, device=self.dev)
        self._ck(self.L.gq_sample_actions(self._p(depth), self._p(gi), self._p(ep), int(seed) & (2 ** 64 - 1), self._p(ei), int(step) & 0xFFFFFFFF, float(fovy),
                                          C.cast(pos, C.c_void_p), C.cast(mat, C.c_void_p), float(z_min), W, H, int(n_rot), int(max_draws), B, self._p(action),
                                          self._p(rnd), self._p(exh), self._stream()), "gq_sample_actions")
        return action, rnd.bool(), exh.bool()

    def greedy(self, q):
        """flat arg-max per image and its split into (pixel index, rotation index) as transform_action does
        (Grasping_Agent_multidiscrete.py:295-299,381-386)"""
        t = self.torch
        B = q.shape[0]
        n = q[0].numel()
        idx = t.empty(B, dtype=t.int32, device=self.dev)
        val = t.empty(B, dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_argmax(self._p(q.contiguous()), B, n, self._p(idx), self._p(val), self._stream()), "gq_argmax")
        hw = q.shape[2] * q.shape[3]
        return t.stack([idx % hw, idx // hw], dim=1), val
