"""QNetLearner: Grasp_Agent.learn() on the device (SURVEY 8f.2) — forward over the batch, gather-BCE loss, backward, Adam, all with the
kernels of libgrasp_qnet.so (csrc/qnet.cu forward + csrc/qnet_learn.cuh backward).  torch is plumbing (buffers, weight repacks).

Reference: Grasping_Agent_multidiscrete.py:388-446
    q_pred = policy_net(state_batch).view(B, -1).gather(1, action_batch)
    loss = F.binary_cross_entropy(q_pred, reward_batch.float());  loss.backward();  optimizer.step();  optimizer.zero_grad()
with optimizer = Adam(policy_net.parameters(), lr, weight_decay=0.00002) (:153-156) and policy_net in training mode, i.e. BatchNorm
normalises over the WHOLE batch here (the acting forward of QNetForward runs the images independently, as the reference does).

Parameters: fp32 masters under the reference's state_dict names (so checkpoints round-trip), bf16 copies in the kernels' layouts
re-packed after every step; activations bf16, pre-BatchNorm outputs fp32, activation gradients bf16, parameter gradients fp32.
Multi-GPU data parallel: pass a torch.distributed process group - the parameter gradients (one flat fp32 buffer, 29.3 MB) are summed
with ONE all-reduce (NCCL over NVLink) between backward and Adam and divided by the world size.

BatchNorm running statistics: every `forward_train` updates the 12 x (running_mean, running_var, num_batches_tracked) buffers as torch's
training-mode forward does (momentum 0.1, unbiased variance; gq_bn_running_update).  With a process group each rank keeps its own
running statistics, from its own shard of the batch; write checkpoints from rank 0, which is what DDP's default broadcast_buffers
amounts to.  The ranks' statistics are not synchronised.

Optimiser: Adam (default) or, with optimizer="sgd", torch.optim.SGD(lr, momentum 0.9, weight_decay) - the reference's OPTIMIZER = "SGD"
(:41,145-152), gq_sgd.  Gradient accumulation (accumulate = K, the reference's NUMBER_ACCUMULATIONS_BEFORE_UPDATE, :27-31,408-446): one
learn_step takes K micro-batches, each with its own training-mode forward and a backward of loss / K; the gradients are summed in order
(gq_grad_accumulate) and one optimizer step follows.  K = 1 with Adam is the single-batch step, kernel for kernel.

Checkpoints in the reference's format (Offline RL/train.py:84-86,147-163, Grasping_Agent_multidiscrete.py:111-158,561-572):
`checkpoint()` -> {"model_state_dict", "optimizer_state_dict"}, `QNetLearner.from_checkpoint(ckpt)` restores parameters, buffers and the
optimiser state (Adam: m, v, step; SGD: the momentum buffers, and the step count from the extra "learner_step" key).  The optimizer part is
produced and read by a CPU torch.optim.Adam / torch.optim.SGD, so its format is torch's own.
"""
import ctypes as C

import numpy as np

from .qnet import _BLOCKS, QNetForward, load_qnet_library, make_torch_qnet

BN_MOMENTUM = 0.1  # nn.BatchNorm2d's default, which Modules.py keeps
_BN_LAYERS = [f"{b}.{bn}" for b in _BLOCKS for bn in ("bn1", "bn2")]


def _meta_qnet():
    """make_torch_qnet(6) without initialising (or drawing random numbers for) its parameters: for the key order and for to_empty()"""
    import torch

    with torch.device("meta"):
        return make_torch_qnet(6)


def model_keys():
    """the 87 state_dict keys of Modules.MULTIDISCRETE_RESNET(6) in order (51 parameters, 36 BatchNorm buffers)"""
    return list(_meta_qnet().state_dict().keys())


def _cpu_qnet():
    import torch

    return _meta_qnet().to_empty(device=torch.device("cpu"))


def adam_to_torch(params, m, v, step, lr, betas, eps, weight_decay):
    """flat Adam state -> torch.optim.Adam(...).state_dict() over make_torch_qnet(6).parameters().  params / m / v: dicts name -> tensor
    (the reference's parameter names), step: the number of steps taken (0: no per-parameter state yet, as torch leaves it)"""
    import torch

    net = _cpu_qnet()
    with torch.no_grad():
        for k, p in net.named_parameters():
            p.copy_(params[k].detach().cpu())
    opt = torch.optim.Adam(net.parameters(), lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay)
    if step > 0:
        for k, p in net.named_parameters():
            opt.state[p] = {"step": torch.tensor(float(step)), "exp_avg": m[k].detach().cpu().clone().to(torch.float32),
                            "exp_avg_sq": v[k].detach().cpu().clone().to(torch.float32)}
    return opt.state_dict()


def adam_from_torch(opt_state):
    """torch.optim.Adam state_dict (over make_torch_qnet(6).parameters()) -> (m, v, step, hyper) with m, v dicts name -> CPU tensor
    (zeros where the optimiser holds no state) and hyper = dict(lr, betas, eps, weight_decay) of its parameter group"""
    import torch

    net = _cpu_qnet()
    with torch.no_grad():
        for p in net.parameters():
            p.zero_()
    opt = torch.optim.Adam(net.parameters())
    opt.load_state_dict(opt_state)
    m, v, steps = {}, {}, set()
    for k, p in net.named_parameters():
        st = opt.state.get(p, {})
        m[k] = st["exp_avg"].detach().clone() if "exp_avg" in st else torch.zeros_like(p)
        v[k] = st["exp_avg_sq"].detach().clone() if "exp_avg_sq" in st else torch.zeros_like(p)
        steps.add(int(float(st["step"])) if "step" in st else 0)
    if len(steps) != 1:
        raise ValueError(f"the optimizer state has different step counts per parameter ({sorted(steps)}); the learner keeps one")
    g = opt.param_groups[0]
    hyper = dict(lr=float(g["lr"]), betas=tuple(float(b) for b in g["betas"]), eps=float(g["eps"]), weight_decay=float(g["weight_decay"]))
    return m, v, steps.pop(), hyper


def sgd_to_torch(params, buf, lr, momentum, weight_decay):
    """flat SGD state -> torch.optim.SGD(lr, momentum, dampening=0, weight_decay, nesterov=False).state_dict() over
    make_torch_qnet(6).parameters().  params / buf: dicts name -> tensor (the reference's parameter names); buf None: no momentum buffer
    yet (before the first step, or momentum = 0), which torch's SGD state then leaves empty"""
    import torch

    net = _cpu_qnet()
    with torch.no_grad():
        for k, p in net.named_parameters():
            p.copy_(params[k].detach().cpu())
    opt = torch.optim.SGD(net.parameters(), lr=lr, momentum=momentum, dampening=0, weight_decay=weight_decay, nesterov=False)
    if buf is not None:
        for k, p in net.named_parameters():
            opt.state[p] = {"momentum_buffer": buf[k].detach().cpu().clone().to(torch.float32)}
    return opt.state_dict()


def sgd_from_torch(opt_state):
    """torch.optim.SGD state_dict (over make_torch_qnet(6).parameters()) -> (buf, hyper): buf a dict name -> CPU tensor of the momentum
    buffers, or None when the optimiser holds none (before its first step, or momentum = 0); hyper = dict(lr, momentum, weight_decay) of
    its parameter group.  A parameter group without the keys newer torch versions added (maximize, foreach, differentiable, fused) loads
    with their defaults.  Nesterov momentum, dampening and maximize are refused: the learner implements none of them."""
    import torch

    g = opt_state["param_groups"][0]
    bad = {k: g.get(k, d) for k, d in (("nesterov", False), ("dampening", 0), ("maximize", False)) if g.get(k, d) != d}
    if bad:
        raise ValueError(f"the SGD state uses {bad}; the learner's SGD has nesterov=False, dampening=0 and maximize=False only")
    net = _cpu_qnet()
    with torch.no_grad():
        for p in net.parameters():
            p.zero_()
    opt = torch.optim.SGD(net.parameters(), lr=1.0)
    opt.load_state_dict(opt_state)
    have = [opt.state.get(p, {}).get("momentum_buffer") for p in net.parameters()]
    if any(b is None for b in have) and any(b is not None for b in have):
        raise ValueError("the optimizer state has momentum buffers for some parameters only; the learner keeps one for all or none")
    buf = None if have[0] is None else {k: b.detach().clone() for (k, _), b in zip(net.named_parameters(), have)}
    g = opt.param_groups[0]
    return buf, dict(lr=float(g["lr"]), momentum=float(g["momentum"]), weight_decay=float(g["weight_decay"]))


def optimizer_of(opt_state):
    """"adam" or "sgd": the optimiser a torch optimizer state_dict belongs to, told by its parameter group (Adam's has betas, SGD's
    momentum and dampening)"""
    g = opt_state["param_groups"][0]
    if "betas" in g:
        return "adam"
    if "momentum" in g and "dampening" in g:
        return "sgd"
    raise ValueError(f"the optimizer state is neither Adam's nor SGD's (parameter group keys {sorted(g)})")


def _bind_learn(L):
    P, I, F = C.c_void_p, C.c_int, C.c_float
    if getattr(L, "_learn_bound", False):
        return L
    L.gq_bn_batch_merge.argtypes = [P, I, I, P]
    L.gq_loss_head_bwd.argtypes = [P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P, P]
    L.gq_bn_relu_bwd.argtypes = [P, P, P, P, P, I, I, I, F, P, P, P, P, P, P, P]
    L.gq_conv_wgrad.argtypes = [P, P, P, P, I, I, I, I, I, I, P]
    L.gq_conv_first_wgrad.argtypes = [P, P, P, P, I, I, I, P]
    L.gq_maxpool_bwd.argtypes = [P, P, P, I, I, I, I, P]
    L.gq_upsample2x_bwd.argtypes = [P, P, I, I, I, I, P]
    L.gq_add_to_bf16.argtypes = [P, P, P, P, C.c_size_t, P]
    L.gq_adam.argtypes = [P, P, P, P, C.c_size_t, F, F, F, F, F, I, P]
    L.gq_sgd.argtypes = [P, P, P, C.c_size_t, F, F, F, I, P]
    L.gq_grad_accumulate.argtypes = [P, P, C.c_size_t, I, P]
    L.gq_bn_running_update.argtypes = [P, P, P, I, I, I, F, P]
    L.gq_loss_head_bwd_weighted.argtypes = [P, P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P, P]
    D, U64 = C.c_double, C.c_uint64
    L.gq_per_push.argtypes = [P, P, P, I, I, P]
    L.gq_per_sample.argtypes = [P, I, C.c_longlong, I, D, U64, U64, C.c_uint32, P, P, P]
    L.gq_per_update.argtypes = [P, P, P, P, P, I, D, D, I, P]
    L._learn_bound = True
    return L


LEARN_SYMBOLS = ["gq_bn_batch_merge", "gq_loss_head_bwd", "gq_bn_relu_bwd", "gq_conv_wgrad", "gq_conv_first_wgrad", "gq_maxpool_bwd", "gq_upsample2x_bwd",
                 "gq_add_to_bf16", "gq_adam", "gq_bn_running_update", "gq_loss_head_bwd_weighted", "gq_per_push", "gq_per_sample", "gq_per_update",
                 "gq_sgd", "gq_grad_accumulate"]
OPTIMIZERS = ("adam", "sgd")


def check_optimizer(optimizer, accumulate, momentum=0.9):
    """-> (optimizer, accumulate, momentum as a float); ValueError unless optimizer is "adam" or "sgd", accumulate (micro-batches per
    update) an int >= 1 and momentum a finite number >= 0"""
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer must be one of {OPTIMIZERS}, not {optimizer!r}")
    if isinstance(accumulate, bool) or not isinstance(accumulate, int) or accumulate < 1:
        raise ValueError(f"accumulate (micro-batches per optimizer step) must be an int >= 1, not {accumulate!r}")
    if isinstance(momentum, bool) or not isinstance(momentum, (int, float)) or not 0.0 <= float(momentum) < float("inf"):
        raise ValueError(f"momentum must be a finite number >= 0, not {momentum!r}")
    return optimizer, accumulate, float(momentum)


class QNetLearner:
    def __init__(self, state_dict=None, device=0, lr=0.001, weight_decay=0.00002, betas=(0.9, 0.999), eps=1e-8, seed=0, process_group=None,
                 optimizer="adam", momentum=0.9, accumulate=1):
        """optimizer: "adam" (torch.optim.Adam(lr, betas, eps, weight_decay)) or "sgd" (torch.optim.SGD(lr, momentum, weight_decay), the
        reference's OPTIMIZER = "SGD"); accumulate = K: every learn_step takes K micro-batches and makes one optimizer step on the sum
        of their gradients, each loss scaled by 1 / K (the reference's NUMBER_ACCUMULATIONS_BEFORE_UPDATE)"""
        import torch

        self.optimizer, self.accumulate, momentum = check_optimizer(optimizer, accumulate, momentum)
        if not torch.cuda.is_available():
            raise RuntimeError("QNetLearner needs a CUDA device (there is no CPU fallback)")
        self.torch = torch
        self.L = _bind_learn(load_qnet_library())
        self.dev = torch.device("cuda", device)
        if state_dict is None:
            torch.manual_seed(seed)
            state_dict = make_torch_qnet(6).state_dict()
        # fp32 masters in ONE flat buffer (Adam and the gradient all-reduce then are single calls); views under the reference's names
        self.names = [k for k, v in state_dict.items() if v.dtype.is_floating_point and "running" not in k]
        sizes = [int(state_dict[k].numel()) for k in self.names]
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        n = int(self.offsets[-1])
        self.flat = torch.empty(n, dtype=torch.float32, device=self.dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=self.dev)
        # optimiser state: Adam's moments, or SGD's momentum buffer (none at momentum 0) and whether its first step has set it
        sgd = self.optimizer == "sgd"
        self.m = None if sgd else torch.zeros(n, dtype=torch.float32, device=self.dev)
        self.v = None if sgd else torch.zeros(n, dtype=torch.float32, device=self.dev)
        self.momentum = momentum
        self.momentum_buf = torch.zeros(n, dtype=torch.float32, device=self.dev) if sgd and self.momentum != 0.0 else None
        self.momentum_init = False
        # the sum of the micro-batches' gradients (accumulate > 1 only; with one micro-batch the optimiser reads `grad`)
        self.grad_acc = torch.zeros(n, dtype=torch.float32, device=self.dev) if self.accumulate > 1 else None
        self.p, self.g = {}, {}
        for k, o, sz in zip(self.names, self.offsets[:-1], sizes):
            shape = tuple(state_dict[k].shape)
            self.p[k] = self.flat[o:o + sz].view(shape)
            self.g[k] = self.grad[o:o + sz].view(shape)
            self.p[k].copy_(state_dict[k].detach().to(self.dev, torch.float32))
        # BatchNorm buffers, torch's initial values (0 / 1 / 0) where the state_dict has none
        self.running_mean, self.running_var, self.num_batches_tracked = {}, {}, {}
        for bn in _BN_LAYERS:
            c = int(state_dict[f"{bn}.weight"].numel())
            rm, rv, nb = (state_dict.get(f"{bn}.{s}") for s in ("running_mean", "running_var", "num_batches_tracked"))
            self.running_mean[bn] = torch.zeros(c, dtype=torch.float32, device=self.dev) if rm is None else rm.detach().to(self.dev, torch.float32).clone()
            self.running_var[bn] = torch.ones(c, dtype=torch.float32, device=self.dev) if rv is None else rv.detach().to(self.dev, torch.float32).clone()
            self.num_batches_tracked[bn] = 0 if nb is None else int(nb)
        self.lr, self.wd, self.betas, self.eps = float(lr), float(weight_decay), betas, float(eps)
        self.step_count = 0
        self.pg = process_group
        self.fw = None
        self.target, self.target_step = None, None  # sync_target()
        self.launches = 0
        self._repack()

    # ------------------------------------------------------------------ parameters
    def state_dict(self):
        """fp32 parameters under the reference's names (parameters only; `model_state_dict()` adds the BatchNorm buffers)"""
        return {k: v.detach().clone() for k, v in self.p.items()}

    def device_state_dict(self):
        """the 51 parameters and 24 BatchNorm running statistics as fp32 tensors on the learner's device, copied device to device, under
        the reference's names (without num_batches_tracked, a host counter): what the eval-mode forward and the target network are
        built from, with no host copy"""
        out = {}
        for k in model_keys():
            bn, _, leaf = k.rpartition(".")
            if k in self.p:
                out[k] = self.p[k].detach().clone()
            elif leaf == "running_mean":
                out[k] = self.running_mean[bn].detach().clone()
            elif leaf == "running_var":
                out[k] = self.running_var[bn].detach().clone()
        return out

    def model_state_dict(self):
        """the full state_dict of Modules.MULTIDISCRETE_RESNET(6): 51 parameters and 36 BatchNorm buffers, CPU fp32 (num_batches_tracked
        int64), in the module's key order - loads with strict=True into the reference's network"""
        t = self.torch
        dev = self.device_state_dict()
        out = {}
        for k in model_keys():
            bn, _, leaf = k.rpartition(".")
            out[k] = t.tensor(self.num_batches_tracked[bn], dtype=t.int64) if leaf == "num_batches_tracked" else dev[k].cpu()
        return out

    def checkpoint(self):
        """{"model_state_dict", "optimizer_state_dict"} as the reference saves them (Offline RL/train.py:147-163); the optimizer part is
        torch.optim.Adam's own state_dict (step, exp_avg = m, exp_avg_sq = v; lr / betas / eps / weight_decay) or, with optimizer="sgd",
        torch.optim.SGD's (momentum_buffer; lr / momentum / dampening 0 / weight_decay / nesterov False).  torch's SGD state has no step
        counter, so an SGD checkpoint also carries "learner_step" (step_count), which torch.load and the reference ignore."""
        if self.optimizer == "sgd":
            buf = self._flat_views(self.momentum_buf) if self.momentum_init else None
            return {"model_state_dict": self.model_state_dict(), "optimizer_state_dict": sgd_to_torch(self.p, buf, self.lr, self.momentum, self.wd),
                    "learner_step": int(self.step_count)}
        return {"model_state_dict": self.model_state_dict(),
                "optimizer_state_dict": adam_to_torch(self.p, self._flat_views(self.m), self._flat_views(self.v), self.step_count, self.lr, self.betas,
                                                      self.eps, self.wd)}

    @classmethod
    def from_checkpoint(cls, ckpt, device=0, **kw):
        """learner from a {"model_state_dict", "optimizer_state_dict"} checkpoint (written by `checkpoint()` or by the reference's scripts):
        parameters, BatchNorm buffers and the optimiser's state.  The optimiser is the checkpoint's: Adam (its parameter group has betas;
        moments and step count restored) or SGD (momentum; momentum buffers restored, step count from "learner_step").  An explicit
        `optimizer=` in `kw` that disagrees is a ValueError.  lr / betas / eps / momentum / weight_decay come from the parameter group
        unless given in `kw`.  A checkpoint without "optimizer_state_dict" starts a fresh optimiser.

        The reference's own SGD checkpoints have no "learner_step": they resume at step_count 0, which restarts what counts learner
        updates - prioritized replay's beta schedule (and its sampling keys) and the phase of the target network's sync period."""
        opt = ckpt.get("optimizer_state_dict")
        if opt is None:
            return cls(ckpt["model_state_dict"], device, **kw)
        kind = optimizer_of(opt)
        if kw.get("optimizer", kind) != kind:
            raise ValueError(f"optimizer={kw['optimizer']!r} was asked for, but the checkpoint holds the state of {kind!r}")
        kw = {**kw, "optimizer": kind}
        if kind == "sgd":
            buf, hyper = sgd_from_torch(opt)
            L = cls(ckpt["model_state_dict"], device, **{**hyper, **kw})
            if buf is not None and L.momentum_buf is not None:
                bv = L._flat_views(L.momentum_buf)
                for k in L.names:
                    bv[k].copy_(buf[k].to(L.dev, L.torch.float32))
                L.momentum_init = True
            L.step_count = int(ckpt.get("learner_step", 0))
            return L
        m, v, step, hyper = adam_from_torch(opt)
        L = cls(ckpt["model_state_dict"], device, **{**hyper, **kw})
        mv, vv = L._flat_views(L.m), L._flat_views(L.v)
        for k in L.names:
            mv[k].copy_(m[k].to(L.dev, L.torch.float32))
            vv[k].copy_(v[k].to(L.dev, L.torch.float32))
        L.step_count = step
        return L

    def _flat_views(self, flat):
        return {k: flat[int(o):int(o) + self.p[k].numel()].view(self.p[k].shape) for k, o in zip(self.names, self.offsets[:-1])}

    def eval_forward(self, max_batch=64):
        """QNetForward in eval mode (batchnorm="running", BatchNorm folded into the weights) from the current parameters and buffers"""
        return QNetForward(self.device_state_dict(), self.dev.index or 0, max_batch=max_batch, batchnorm="running")

    def sync_target(self, max_batch=64):
        """target network := the eval-mode forward of the current parameters and running statistics (the reference's
        target_net.load_state_dict(policy_net.state_dict()) with target_net.eval(), Grasping_Agent_multidiscrete.py:105-115,410-413).
        It is a separate copy: the learner's later steps do not change it.  Sets `target` and `target_step` (the step_count it was
        built at); neither is part of a checkpoint."""
        self.target = self.eval_forward(max_batch)
        self.target_step = self.step_count
        return self.target

    def _repack(self):
        """bf16 kernel layouts from the fp32 masters: the forward's [Cout][kh][kw][Cin] (QNetForward) and, for the input-gradient
        convolutions, the spatially flipped in/out-transposed [Cin][kh][kw][Cout]"""
        t = self.torch
        sd = {k: v for k, v in self.p.items()}
        if self.fw is None:
            self.fw = QNetForward(sd, self.dev.index or 0, max_batch=1 << 30)
        else:
            fresh = QNetForward(sd, self.dev.index or 0, max_batch=1 << 30)
            fresh.launches = self.fw.launches
            self.fw = fresh
        self.wT = []
        for name in _BLOCKS:
            d = {}
            for c in ("conv1", "conv2", "conv3"):
                w = self.p[f"{name}.{c}.weight"]  # [Cout, Cin, kh, kw]
                d[c] = w.flip(2, 3).permute(1, 2, 3, 0).contiguous().to(t.bfloat16)
            self.wT.append(d)

    # ------------------------------------------------------------------ small helpers
    def _ck(self, r, what):
        if r != 0:
            raise RuntimeError(f"{what} failed ({r}): {self.L.gq_last_error().decode()}")
        self.launches += 1

    def _p(self, x):
        return None if x is None else C.c_void_p(x.data_ptr())

    def _st(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.dev).cuda_stream)

    def _merge(self, stats, B, Cc):
        self._ck(self.L.gq_bn_batch_merge(self._p(stats), B, Cc, self._st()), "gq_bn_batch_merge")

    def _running_update(self, bn, stats, B, HW, Cc):
        """torch's training-mode buffer update of BatchNorm layer `bn` from its merged batch statistics"""
        self._ck(self.L.gq_bn_running_update(self._p(stats), self._p(self.running_mean[bn]), self._p(self.running_var[bn]), B, HW, Cc, BN_MOMENTUM, self._st()),
                 "gq_bn_running_update")
        self.num_batches_tracked[bn] += 1

    # ------------------------------------------------------------------ forward over the batch (training mode), activations kept
    def _block_fwd(self, x, blk, B, H, W, name):
        fw = self.fw
        cin, cout = blk["cin"], blk["cout"]
        o1, s1 = fw.conv_tc(x, blk["w1"], None, B, H, W, cin, cout, 3, True)
        self._merge(s1, B, cout)
        self._running_update(f"{name}.bn1", s1, B, H * W, cout)
        a1 = fw.bn_act(o1, s1, blk["g1"], blk["be1"], None, B, H * W, cout)
        o2, s2 = fw.conv_tc(a1, blk["w2"], None, B, H, W, cout, cout, 3, True)
        self._merge(s2, B, cout)
        self._running_update(f"{name}.bn2", s2, B, H * W, cout)
        out = fw.conv_tc_block_out(x, blk["w3"], blk["b3"], o2, s2, blk["g2"], blk["be2"], B, H, W, cin, cout, 1)
        return out, dict(x=x, o1=o1, s1=s1, a1=a1, o2=o2, s2=s2, out=out, H=H, W=W)

    def forward_train(self, state):
        """state [B,4,H,W] f32 -> (q [B,A,H,W] f32, saved activations).  Updates the BatchNorm running statistics, as torch's
        training-mode forward does."""
        t, fw = self.torch, self.fw
        state = state.to(self.dev, t.float32).contiguous()
        B, _, H, W = state.shape
        x0 = t.empty((B, H, W, 64), dtype=t.bfloat16, device=self.dev)
        fw._ck(fw.L.gq_conv_first(fw._p(state), fw._p(fw.w_first), fw._p(x0), B, H, W, fw._stream()), "gq_conv_first")
        h, w = (H + 1) // 2, (W + 1) // 2
        p0 = fw.maxpool(x0, B, H, W, 64)
        b0, sv0 = self._block_fwd(p0, fw.blocks[0], B, h, w, _BLOCKS[0])
        h2, w2 = (h + 1) // 2, (w + 1) // 2
        p1 = fw.maxpool(b0.view(B, h, w, 128), B, h, w, 128)
        b1, sv1 = self._block_fwd(p1, fw.blocks[1], B, h2, w2, _BLOCKS[1])
        b2, sv2 = self._block_fwd(b1, fw.blocks[2], B, h2, w2, _BLOCKS[2])
        b3, sv3 = self._block_fwd(b2, fw.blocks[3], B, h2, w2, _BLOCKS[3])
        b4, sv4 = self._block_fwd(b3, fw.blocks[4], B, h2, w2, _BLOCKS[4])
        u0 = fw.upsample(b4.view(B, h2, w2, 128), B, h2, w2, 128)
        b5, sv5 = self._block_fwd(u0, fw.blocks[5], B, 2 * h2, 2 * w2, _BLOCKS[5])
        A = fw.A
        q = t.empty((B, A, 4 * h2, 4 * w2), dtype=t.float32, device=self.dev)
        z = t.empty((B, A, 2 * h2, 2 * w2), dtype=t.float32, device=self.dev)
        fw._ck(fw.L.gq_head_up2(fw._p(b5), fw._p(fw.w_head), fw._p(fw.b_head), fw._p(z), fw._p(q), B, 2 * h2, 2 * w2, A, fw._stream()), "gq_head_up2")
        saved = dict(state=state, x0=x0, b0=b0, b5=b5, blocks=[sv0, sv1, sv2, sv3, sv4, sv5], dims=(B, H, W, h, w, h2, w2))
        return q, saved

    # ------------------------------------------------------------------ backward
    def _bn_relu_bwd(self, dY, act, o, stats, gamma, B, HW, Cc, want_dpre, gname, bname):
        t = self.torch
        d_o = t.empty((B, HW, Cc), dtype=t.bfloat16, device=self.dev)
        dpre = t.empty((B, HW, Cc), dtype=t.bfloat16, device=self.dev) if want_dpre else None
        part = t.empty(((B * HW + 127) // 128) * Cc * 2, dtype=t.float32, device=self.dev)
        sums = t.empty(2 * Cc, dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_bn_relu_bwd(self._p(dY), self._p(act), self._p(o), self._p(stats), self._p(gamma), B, HW, Cc, 1e-5, self._p(dpre), self._p(part),
                                       self._p(sums), self._p(self.g[gname]), self._p(self.g[bname]), self._p(d_o), self._st()), "gq_bn_relu_bwd")
        return d_o, dpre

    def _wgrad(self, dY, x, B, H, W, cin, cout, ks, name):
        t = self.torch
        part = t.empty(B * cout * ks * ks * cin, dtype=t.float32, device=self.dev)
        dW = t.empty((cout, ks * ks, cin), dtype=t.float32, device=self.dev)  # kernel layout [Cout][taps][Cin]
        self._ck(self.L.gq_conv_wgrad(self._p(dY), self._p(x), self._p(part), self._p(dW), B, H, W, cin, cout, ks, self._st()), "gq_conv_wgrad")
        self.g[name].copy_(dW.view(cout, ks, ks, cin).permute(0, 3, 1, 2))  # -> the reference's [Cout, Cin, kh, kw]

    def _dgrad(self, dY, wT, B, H, W, cin_of_conv, cout_of_conv, ks):
        """gradient w.r.t. the input of a convolution = the forward convolution of dY with the flipped / transposed weights"""
        y, _ = self.fw.conv_tc(dY, wT, None, B, H, W, cout_of_conv, cin_of_conv, ks, False)
        return y  # f32 [B,H,W,Cin]

    def _to_bf16(self, a, b=None, c_bf16=None):
        t = self.torch
        out = t.empty(a.shape, dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_add_to_bf16(self._p(a), self._p(b), self._p(c_bf16), self._p(out), a.numel(), self._st()), "gq_add_to_bf16")
        return out

    def _block_bwd(self, i, sv, dOut, B):
        """BasicBlock backward (Modules.py:128-142): dOut [B,HW,Cout] bf16 -> dX [B,HW,Cin] bf16; parameter gradients into self.g"""
        name, blk, wT = _BLOCKS[i], self.fw.blocks[i], self.wT[i]
        cin, cout, H, W = blk["cin"], blk["cout"], sv["H"], sv["W"]
        HW = H * W
        # out = relu(bn2(o2) + conv3(x) + b3)
        d_o2, dpre = self._bn_relu_bwd(dOut, sv["out"], sv["o2"], sv["s2"], blk["g2"], B, HW, cout, True, f"{name}.bn2.weight", f"{name}.bn2.bias")
        self.g[f"{name}.conv3.bias"].copy_(self.g[f"{name}.bn2.bias"])  # both are sum(dpre) over batch and pixels
        self._wgrad(dpre, sv["x"], B, H, W, cin, cout, 1, f"{name}.conv3.weight")
        dx_short = self._dgrad(dpre, wT["conv3"], B, H, W, cin, cout, 1)
        # o2 = conv2(a1)
        self._wgrad(d_o2, sv["a1"], B, H, W, cout, cout, 3, f"{name}.conv2.weight")
        d_a1 = self._to_bf16(self._dgrad(d_o2, wT["conv2"], B, H, W, cout, cout, 3))
        # a1 = relu(bn1(o1)), o1 = conv1(x)
        d_o1, _ = self._bn_relu_bwd(d_a1, sv["a1"], sv["o1"], sv["s1"], blk["g1"], B, HW, cout, False, f"{name}.bn1.weight", f"{name}.bn1.bias")
        self._wgrad(d_o1, sv["x"], B, H, W, cin, cout, 3, f"{name}.conv1.weight")
        dx_main = self._dgrad(d_o1, wT["conv1"], B, H, W, cin, cout, 3)
        return self._to_bf16(dx_main, dx_short)

    # parameter groups in the order the backward pass completes them (each one contiguous in the flat buffers)
    GROUPS = ("1.C1.", "1.RB3.", "1.RB2.", "1.RB1.", "0.RB3.", "0.RB2.", "0.RB1.", "0.C1.")

    def grad_slice(self, prefix, flat=None):
        """the contiguous piece of the flat gradient buffer (or of `flat`, laid out alike) that holds every parameter whose name starts
        with `prefix`"""
        idx = [i for i, k in enumerate(self.names) if k.startswith(prefix)]
        assert idx and idx == list(range(idx[0], idx[-1] + 1)), prefix
        return (self.grad if flat is None else flat)[int(self.offsets[idx[0]]):int(self.offsets[idx[-1] + 1])]

    def backward(self, q, saved, action, reward, on_ready=None, weight=None):
        """-> loss (0-dim tensor), q_pred [B]; fills self.grad (every parameter gradient of the step).  `on_ready(prefix)` is called as
        soon as all gradients of one parameter group (a BasicBlock, the head, the first convolution) have been enqueued - the
        multi-GPU learner starts that group's all-reduce there, under the rest of the backward pass.  weight [B] f32 on the device
        (prioritized replay's importance weights): the loss is binary_cross_entropy(q_pred, reward, weight=weight)."""
        ready = on_ready if on_ready is not None else (lambda prefix: None)
        t, fw = self.torch, self.fw
        B, H, W, h, w, h2, w2 = saved["dims"]
        A = fw.A
        action = action.to(self.dev, t.int64).reshape(B).contiguous()
        reward = reward.to(self.dev, t.float32).reshape(B).contiguous()
        loss_terms = t.empty(B, dtype=t.float32, device=self.dev)
        qsel = t.empty(B, dtype=t.float32, device=self.dev)
        d_b5 = t.empty((B, 2 * h2 * 2 * w2, 64), dtype=t.bfloat16, device=self.dev)
        dWp = t.empty((B, A, 64), dtype=t.float32, device=self.dev)
        dbp = t.empty((B, A), dtype=t.float32, device=self.dev)
        dW_head = t.empty((A, 64), dtype=t.float32, device=self.dev)
        if weight is None:
            self._ck(self.L.gq_loss_head_bwd(self._p(q), self._p(saved["b5"]), self._p(fw.w_head), self._p(action), self._p(reward), B, A, 2 * h2, 2 * w2,
                                             self._p(loss_terms), self._p(qsel), self._p(d_b5), self._p(dWp), self._p(dbp), self._p(dW_head), self._p(self.g["1.C1.bias"]),
                                             self._st()), "gq_loss_head_bwd")
        else:
            weight = weight.to(self.dev, t.float32).reshape(B).contiguous()
            self._ck(self.L.gq_loss_head_bwd_weighted(self._p(q), self._p(saved["b5"]), self._p(fw.w_head), self._p(action), self._p(reward), self._p(weight), B, A,
                                                      2 * h2, 2 * w2, self._p(loss_terms), self._p(qsel), self._p(d_b5), self._p(dWp), self._p(dbp), self._p(dW_head),
                                                      self._p(self.g["1.C1.bias"]), self._st()), "gq_loss_head_bwd_weighted")
        self.g["1.C1.weight"].copy_(dW_head.view(A, 64, 1, 1))
        ready("1.C1.")
        sv = saved["blocks"]
        d_u0 = self._block_bwd(5, sv[5], d_b5, B)                                   # 1.RB3 @100x100
        ready("1.RB3.")
        d_b4 = t.empty((B, h2 * w2, 128), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_upsample2x_bwd(self._p(d_u0), self._p(d_b4), B, h2, w2, 128, self._st()), "gq_upsample2x_bwd")
        d = self._block_bwd(4, sv[4], d_b4, B)                                      # 1.RB2
        ready("1.RB2.")
        d = self._block_bwd(3, sv[3], d, B)                                         # 1.RB1
        ready("1.RB1.")
        d = self._block_bwd(2, sv[2], d, B)                                         # 0.RB3
        ready("0.RB3.")
        d_p1 = self._block_bwd(1, sv[1], d, B)                                      # 0.RB2 @50x50
        ready("0.RB2.")
        d_b0 = t.empty((B, h * w, 128), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_maxpool_bwd(self._p(saved["b0"]), self._p(d_p1), self._p(d_b0), B, h, w, 128, self._st()), "gq_maxpool_bwd")
        d_p0 = self._block_bwd(0, sv[0], d_b0, B)                                   # 0.RB1 @100x100
        ready("0.RB1.")
        d_x0 = t.empty((B, H * W, 64), dtype=t.bfloat16, device=self.dev)
        self._ck(self.L.gq_maxpool_bwd(self._p(saved["x0"]), self._p(d_p0), self._p(d_x0), B, H, W, 64, self._st()), "gq_maxpool_bwd")
        n = B * H * W
        part = t.empty(((n + 2047) // 2048) * 64 * 36, dtype=t.float32, device=self.dev)
        dWf = t.empty((64, 9, 4), dtype=t.float32, device=self.dev)
        self._ck(self.L.gq_conv_first_wgrad(self._p(d_x0), self._p(saved["state"]), self._p(part), self._p(dWf), B, H, W, self._st()), "gq_conv_first_wgrad")
        self.g["0.C1.weight"].copy_(dWf.view(64, 3, 3, 4).permute(0, 3, 1, 2))
        ready("0.C1.")
        return loss_terms.mean(), qsel

    # ------------------------------------------------------------------ one learn() call
    def learn_step(self, state, action, reward, return_pred=False, weight=None):
        """state [B,4,H,W] f32 (what the agent stores in its replay buffer), action [B] or [B,1] flat indices rot*H*W + y*W + x, reward [B] or
        [B,1].  Returns the loss as a float (one device->host read, like the reference's `loss.item()`); with return_pred=True
        (loss, q_pred [B] on the device), q_pred being the gathered Q-values of the training forward (Offline RL/train.py:109,122).
        weight: None (the reference's loss) or [B] f32 importance weights on the device; the step then minimises and returns the
        weighted loss binary_cross_entropy(q_pred, reward, weight=weight).

        With accumulate = K the B rows (B divisible by K) are K micro-batches of B / K consecutive rows, as the reference's learn() slices
        its BATCH_SIZE = K * MAX_POSSIBLE_SAMPLES draw: each one gets its own training-mode forward (its own BatchNorm statistics and one
        running-statistics update) and a backward of its loss / K (weights w_b / K, w_b = 1 without importance weights), the gradients
        are summed in micro-batch order (gq_grad_accumulate), then one optimizer step.  The loss returned is the sum of the scaled
        losses, i.e. the mean of the micro-batch losses; q_pred holds all B gathered Q-values in row order."""
        t = self.torch
        K = self.accumulate
        B = int(state.shape[0])
        if B % K:
            raise ValueError(f"learn_step: {B} rows do not split into accumulate = {K} equal micro-batches")
        if K == 1:  # (the arguments as given: no slicing on the single-batch path)
            micro = [(state, action, reward, weight)]
        else:
            b = B // K
            action, reward = action.reshape(B), reward.reshape(B)
            wb = t.ones(B, dtype=t.float32, device=self.dev) if weight is None else weight.to(self.dev, t.float32).reshape(B)
            weight = wb / K
            micro = [(state[k * b:(k + 1) * b], action[k * b:(k + 1) * b], reward[k * b:(k + 1) * b], weight[k * b:(k + 1) * b]) for k in range(K)]
        works, losses, qsels = [], [], []
        for k, (s, a, r, w) in enumerate(micro):
            q, saved = self.forward_train(s)
            on_ready = None
            if K > 1 or self.pg is not None:
                on_ready = self._on_ready(works, first=k == 0, reduce=k == K - 1)
            loss, qsel = self.backward(q, saved, a, r, on_ready, w)
            losses.append(loss)
            qsels.append(qsel)
        for work in works:
            work.wait()  # (stream-level wait: the optimizer step below is ordered after the last piece)
        self.step_count += 1
        self._optimizer_step(self.grad if K == 1 else self.grad_acc)
        self._repack()
        loss = losses[0] if K == 1 else t.stack(losses).sum()
        qsel = qsels[0] if K == 1 else t.cat(qsels)
        return (float(loss), qsel) if return_pred else float(loss)

    def _on_ready(self, works, first, reduce):
        """the per-parameter-group hook of one micro-batch's backward: with accumulate > 1 the group's gradient is added into grad_acc,
        and on the last micro-batch (`reduce`) with a process group the group's summed gradient is averaged over the ranks"""
        dist = None
        if self.pg is not None and reduce:
            import torch.distributed as dist

        def on_ready(prefix):
            g = self.grad_slice(prefix)
            if self.accumulate > 1:
                acc = self.grad_slice(prefix, self.grad_acc)
                self._ck(self.L.gq_grad_accumulate(self._p(acc), self._p(g), g.numel(), int(first), self._st()), "gq_grad_accumulate")
                g = acc
            if dist is not None:
                # the learner's one collective: the 29.3 MB of fp32 gradients averaged over the ranks, issued per parameter group (8 pieces,
                # last layers first) on NCCL's stream as soon as the group's last wgrad kernel is enqueued, so that the transfer of the
                # 512/256-channel blocks runs under the backward pass of the layers in front of them (Grasping_Agent_multidiscrete.py has a
                # single process; this is north_star's "gradient/batch reduction").  With accumulation: once per optimizer step, the sum.
                works.append(dist.all_reduce(g, op=dist.ReduceOp.AVG, group=self.pg, async_op=True))

        return on_ready

    def _optimizer_step(self, grad):
        """one step of the learner's optimiser on the flat gradient `grad` (step_count already counts it)"""
        if self.optimizer == "adam":
            self._ck(self.L.gq_adam(self._p(self.flat), self._p(grad), self._p(self.m), self._p(self.v), self.flat.numel(), self.lr, self.betas[0],
                                    self.betas[1], self.eps, self.wd, self.step_count, self._st()), "gq_adam")
            return
        self._ck(self.L.gq_sgd(self._p(self.flat), self._p(grad), self._p(self.momentum_buf), self.flat.numel(), self.lr, self.momentum, self.wd,
                               int(not self.momentum_init), self._st()), "gq_sgd")
        self.momentum_init = self.momentum_buf is not None
