"""Learner BasicBlocks one at a time against float64 autograd, at the network's real shapes and the batch sizes it trains with.

QNetLearner._block_fwd / _block_bwd chain batch-merged BatchNorm statistics (gq_bn_batch_merge), the BatchNorm backward with its 1/(B*HW),
the shortcut gradient dpre, the conv3.bias copy, dgrad through the flipped / transposed weights, split-K weight gradients over the
images, and bf16 hand-offs in between.  The whole-network test (test_qnet_learn.py) has to be loose because the loss touches one pixel
per image; here every block gets a dense incoming gradient and a float64 oracle that rounds to bf16 exactly where the kernels do:

    forward:  x bf16 (input); o1 = conv1(x), o2 = conv2(a1) full precision; a1 = bf16(relu(bn1(o1))); out = bf16(relu(bn2(o2) + conv3(x) + b3))
    backward: dOut bf16 (input); dpre = dOut * (out > 0) (exact); d_o2, d_a1, d_o1 rounded to bf16; dX = bf16(dx_main + dx_short);
              weight / gamma / beta / bias gradients not rounded

With the rounding points matched the two sides differ by fp32 accumulation, occasional one-ulp bf16 flips and the ReLU decisions those
flips move (see BOUND); a second run of the oracle with the learner's a1 and ReLU masks takes the latter out and bounds the rest tightly.
The oracle itself is pinned on CPU (rounding off) to the reference module's BasicBlock in train() mode.
"""
import pytest
import torch
import torch.nn.functional as F

from mujoco_rl_ur5_b200.qnet import _BLOCKS, BN_EPS

gpu = pytest.mark.gpu
BATCHES = (1, 12, 15)  # one image; the reference's BATCH_SIZE (the bench's learn leg); the offline trainer's batch
PARAMS = ("conv1.weight", "bn1.weight", "bn1.bias", "conv2.weight", "bn2.weight", "bn2.bias", "conv3.weight", "conv3.bias")
CONV_WEIGHTS = ("conv1.weight", "conv2.weight", "conv3.weight")  # the learner packs these as bf16; gamma, beta and bias stay fp32


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


class _Round(torch.autograd.Function):
    """identity whose forward value (fwd) and / or backward gradient (bwd) is rounded to bf16; with `value` given the forward returns that
    tensor instead, and the gradient still flows to the input as through an identity"""

    @staticmethod
    def forward(ctx, t, fwd, bwd, value=None):
        ctx.bwd = bwd
        if value is not None:
            return value.clone()
        return t.to(torch.bfloat16).to(t.dtype) if fwd else t.clone()

    @staticmethod
    def backward(ctx, g):
        return (g.to(torch.bfloat16).to(g.dtype) if ctx.bwd else g), None, None, None


def oracle_block(x, p, d_out, rounding, learner_fwd=None):
    """BasicBlock.forward (Modules.py:128-142) with training-mode BatchNorm over the whole batch, in the dtype of `x`, then backward of
    `d_out`.  x [B,Cin,H,W] and the tensors of `p` (keys PARAMS) are autograd leaves; rounding=True rounds to bf16 where the learner's
    kernels do.  learner_fwd = dict(a1, out) of the learner (with rounding): a1 is that tensor and both ReLU masks are the learner's,
    which takes the one-ulp flips of a1 and the ReLU decisions they cause out of the comparison of everything else.
    -> dict(o1, a1, o2, out) of the forward; x.grad and p[k].grad hold the gradients."""
    r = (lambda t, fwd, bwd, value=None: _Round.apply(t, fwd, bwd, value)) if rounding else (lambda t, fwd, bwd, value=None: t)
    lf = learner_fwd or {}
    relu = lambda t, k: t * (lf[k] > 0) if k in lf else F.relu(t)
    xi = r(x, False, True)  # both branches' gradients meet here and are rounded once
    o1 = r(F.conv2d(xi, p["conv1.weight"], padding=1), False, True)
    a1 = r(relu(F.batch_norm(o1, None, None, p["bn1.weight"], p["bn1.bias"], True, 0.0, BN_EPS), "a1"), True, True, lf.get("a1"))
    o2 = r(F.conv2d(a1, p["conv2.weight"], padding=1), False, True)
    out = relu(F.batch_norm(o2, None, None, p["bn2.weight"], p["bn2.bias"], True, 0.0, BN_EPS) + F.conv2d(xi, p["conv3.weight"], p["conv3.bias"]), "out")
    out = r(out, True, False)
    out.backward(d_out)
    return dict(o1=o1.detach(), a1=a1.detach(), o2=o2.detach(), out=out.detach())


def _batch_moments(o):
    """batch mean and biased / unbiased variance per channel of o [B,C,H,W] (what BatchNorm normalises with / stores)"""
    return o.mean(dim=(0, 2, 3)), o.var(dim=(0, 2, 3), unbiased=False), o.var(dim=(0, 2, 3), unbiased=True)


# ------------------------------------------------------------------------------------------------ CPU: the oracle is the reference's block
def test_oracle_without_rounding_is_the_reference_basic_block():
    """rounding off, float64: outputs, input gradient, all eight parameter gradients and the running-statistics update equal torch autograd
    of make_torch_qnet's BasicBlock (0.RB1, 64 -> 128) in train() mode"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    torch.manual_seed(0)
    blk = make_torch_qnet(6)[0].RB1.double().train()
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():  # gamma, beta away from torch's 1 / 0, so that a lost gamma or beta term shows
        for bn in (blk.bn1, blk.bn2):
            bn.weight.copy_(torch.rand(bn.weight.shape, generator=g, dtype=torch.float64) + 0.5)
            bn.bias.copy_(torch.randn(bn.bias.shape, generator=g, dtype=torch.float64) * 0.2)
    B, H, W = 2, 10, 12
    x = torch.rand((B, 64, H, W), generator=g, dtype=torch.float64)
    d_out = torch.randn((B, 128, H, W), generator=g, dtype=torch.float64)
    xm = x.clone().requires_grad_(True)
    ym = blk(xm)
    ym.backward(d_out)
    xo = x.clone().requires_grad_(True)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in blk.named_parameters()}
    assert set(p) == set(PARAMS)
    f = oracle_block(xo, p, d_out, rounding=False)
    tight = dict(rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(f["out"], ym.detach(), **tight)
    torch.testing.assert_close(xo.grad, xm.grad, **tight)
    for k, v in blk.named_parameters():
        torch.testing.assert_close(p[k].grad, v.grad, **tight, msg=k)
    # BatchNorm2d's buffers after one training forward from (0, 1): momentum 0.1 towards the batch mean and the UNBIASED variance
    with torch.no_grad():
        o1 = F.conv2d(x, blk.conv1.weight, padding=1)
        a1 = F.relu(F.batch_norm(o1, None, None, blk.bn1.weight, blk.bn1.bias, True, 0.0, BN_EPS))
        o2 = F.conv2d(a1, blk.conv2.weight, padding=1)
    for o, bn in ((o1, blk.bn1), (o2, blk.bn2)):
        mean, _, var_u = _batch_moments(o)
        torch.testing.assert_close(bn.running_mean, 0.1 * mean, **tight)
        torch.testing.assert_close(bn.running_var, 0.9 + 0.1 * var_u, **tight)
    torch.testing.assert_close(f["o1"], o1, **tight)
    torch.testing.assert_close(f["o2"], o2, **tight)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def learner():
    """QNetLearner on make_torch_qnet(6) with seed 0, BatchNorm gamma in [0.5, 1.5) and beta ~ N(0, 0.2) instead of torch's 1 / 0"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    torch.manual_seed(0)
    sd = {k: v.clone() for k, v in make_torch_qnet(6).state_dict().items()}
    g = torch.Generator().manual_seed(11)
    for k in sd:
        if ".bn" in k and k.endswith(".weight"):
            sd[k] = torch.rand(sd[k].shape, generator=g) + 0.5
        elif ".bn" in k and k.endswith(".bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.2
    return QNetLearner(sd, 0)


@pytest.fixture(scope="module", params=BATCHES, ids=lambda b: f"B{b}")
def train_forward(request, learner):
    """one forward_train of the learner on B torch.rand states (as the bench feeds it): the blocks' real activations, and the running
    statistics before and after"""
    B = request.param
    snap = lambda: {k: (learner.running_mean[k].clone(), learner.running_var[k].clone()) for k in learner.running_mean}
    before = snap()
    state = torch.rand((B, 4, 200, 200), generator=torch.Generator().manual_seed(100 + B))
    _, saved = learner.forward_train(state)
    torch.cuda.synchronize()
    return B, saved, before, snap()


# Relative L2 errors, bound = the largest value measured over the six blocks and B = 1, 12, 15 on an H100 80GB HBM3 (700 W) times at most 3
# (measured maximum in the comment).
#
# BOUND: against the rounded oracle, independent of the learner.  Both sides round a1 = relu(bn1(o1)) to bf16, one from fp32 and one from
# float64: where those straddle a rounding boundary they differ by one ulp, which moves o2 by ~5e-5.  That flips the ReLU mask of `out`
# wherever bn2(o2) + conv3(x) + b3 is that close to 0 (up to 2e-5 of the elements), and each flip adds or removes a whole dOut value, so
# every gradient of the block moves by ~sqrt(flip fraction) = a few 1e-3.
BOUND = {
    "o1": 1e-5,                              # fp32 convolution output (3.4e-6)
    "a1": 2.5e-4,                            # bf16, one-ulp flips (8.4e-5)
    "o2": 2e-4,                              # fp32, on the oracle's own a1 (8.5e-5)
    "stats1": 1.2e-5, "stats2": 1.2e-5,      # merged (sum, sum of squares) / B (5.0e-6)
    "var1": 1.5e-5, "var2": 1.5e-5,          # the fp32 variance E[o^2] - mean^2 the kernels normalise with (6.5e-6)
    "running_mean1": 1e-5, "running_mean2": 1e-5,  # (3.7e-6)
    "running_var1": 3e-7, "running_var2": 3e-7,    # (1.2e-7)
    "out": 1e-3,                             # bf16 (4.1e-4)
    "out-mask flips": 6e-5,                  # fraction of elements (2.0e-5)
    "dX": 1.5e-2, "conv1.weight": 1.5e-2, "conv2.weight": 1.5e-2, "conv3.weight": 1.5e-2, "conv3.bias": 1.5e-2,  # (6.1e-3, the mask flips)
    "bn1.weight": 1.5e-2, "bn1.bias": 1.5e-2, "bn2.weight": 1.5e-2, "bn2.bias": 1.5e-2,
}
# BOUND_FORCED: against the rounded oracle run with the learner's a1 and the learner's two ReLU masks (learner_fwd).  What is left is fp32
# accumulation and one-ulp flips at the rounded gradients d_o2, d_a1, d_o1.  bn2 and conv3.bias see only dpre = dOut * mask (exact) and
# fp32 sums.
BOUND_FORCED = {
    "o2": 1e-5, "out": 2e-4,                 # (3.4e-6, 7.8e-5)
    "dX": 4e-3,                              # (1.5e-3)
    "conv1.weight": 2e-3, "bn1.weight": 2e-3, "bn1.bias": 2e-3,  # (7.4e-4, 6.7e-4, 8.0e-4)
    "conv2.weight": 4e-4,                    # (1.6e-4)
    "conv3.weight": 2.5e-5,                  # (9.6e-6)
    "bn2.weight": 5e-6, "bn2.bias": 1e-7, "conv3.bias": 1e-7,  # (1.8e-6, 3.0e-8, 3.0e-8)
}
# LOOSE: against the oracle WITHOUT bf16 rounding, what the rounding points cost (5.8e-2)
LOOSE = 0.1


@gpu
@pytest.mark.parametrize("i", range(6), ids=_BLOCKS)
def test_block_matches_float64(learner, train_forward, i):
    B, saved, before, after = train_forward
    name, blk, sv = _BLOCKS[i], learner.fw.blocks[i], saved["blocks"][i]
    cin, cout, H, W = blk["cin"], blk["cout"], sv["H"], sv["W"]
    nchw = lambda t, c: t.reshape(B, H, W, c).permute(0, 3, 1, 2).double()
    g = torch.Generator(device="cuda").manual_seed(1000 * B + i)
    d_out = torch.randn((B, H * W, cout), generator=g, device="cuda").to(torch.bfloat16)
    dX = learner._block_bwd(i, sv, d_out, B)
    torch.cuda.synchronize()
    ours = {k: learner.g[f"{name}.{k}"].clone() for k in PARAMS}
    ours["dX"] = nchw(dX, cin)
    fwd = {k: nchw(sv[k], cout) for k in ("o1", "a1", "o2", "out")}
    GRADS = ("dX",) + PARAMS

    def oracle(rounding, learner_fwd=None):
        x = nchw(sv["x"], cin).requires_grad_(True)
        p = {k: (learner.p[f"{name}.{k}"].to(torch.bfloat16) if k in CONV_WEIGHTS else learner.p[f"{name}.{k}"]).double().clone().requires_grad_(True)
             for k in PARAMS}
        f = oracle_block(x, p, nchw(d_out, cout), rounding, learner_fwd)
        return f, dict({k: v.grad for k, v in p.items()}, dX=x.grad)

    f, grads = oracle(True)
    err = {k: rel(fwd[k], f[k]) for k in ("o1", "a1", "o2", "out")}
    HW = H * W
    for j in (1, 2):
        o, s = f[f"o{j}"], sv[f"s{j}"]  # s [B, C, 2]: after the merge every image's row holds the batch totals / B
        mean, var, var_u = _batch_moments(o)
        s_ref = torch.stack([o.sum(dim=(0, 2, 3)), (o * o).sum(dim=(0, 2, 3))], dim=1) / B
        err[f"stats{j}"] = rel(s, s_ref.expand(B, cout, 2))
        m32 = s[0, :, 0] / HW
        err[f"var{j}"] = rel(s[0, :, 1] / HW - m32 * m32, var)
        bn = f"{name}.bn{j}"
        err[f"running_mean{j}"] = rel(after[bn][0], 0.9 * before[bn][0].double() + 0.1 * mean)
        err[f"running_var{j}"] = rel(after[bn][1], 0.9 * before[bn][1].double() + 0.1 * var_u)
    err.update({k: rel(ours[k], grads[k]) for k in GRADS})
    err["out-mask flips"] = float(((fwd["out"] > 0) != (f["out"] > 0)).double().mean())
    fa, grads_a = oracle(True, dict(a1=fwd["a1"], out=fwd["out"]))
    err_a = {k: rel(fwd[k], fa[k]) for k in ("o2", "out")}
    err_a.update({k: rel(ours[k], grads_a[k]) for k in GRADS})
    f0, grads0 = oracle(False)
    loose = {k: rel(fwd[k], f0[k]) for k in ("o1", "o2", "out")}
    loose.update({k: rel(ours[k], grads0[k]) for k in GRADS})
    print(f"\n{name} B={B}: " + "  ".join(f"{k} {v:.2e}" for k, v in err.items()))
    print(f"{name} B={B} learner's a1 and masks: " + "  ".join(f"{k} {v:.2e}" for k, v in err_a.items()))
    print(f"{name} B={B} unrounded oracle: " + "  ".join(f"{k} {v:.2e}" for k, v in loose.items()))
    bad = {k: (v, BOUND[k]) for k, v in err.items() if not v <= BOUND[k]}
    bad.update({"learner's a1 and masks: " + k: (v, BOUND_FORCED[k]) for k, v in err_a.items() if not v <= BOUND_FORCED[k]})
    bad.update({"unrounded: " + k: (v, LOOSE) for k, v in loose.items() if not v <= LOOSE})
    assert not bad, bad
