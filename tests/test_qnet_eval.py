"""Eval-mode Q-network: BatchNorm running statistics in the learner (gq_bn_running_update), the BN-folded wgmma forward
(gq_conv_tc_fused, QNetForward(batchnorm="running")) and reference-format checkpoints (QNetLearner.checkpoint / from_checkpoint).

Bars as in tests/test_qnet.py: one convolution within bf16 output rounding + summation order of F.conv2d on the same bf16 operands;
the whole network within mean |err| 5e-3, max 5e-2 of the fp32 torch module, greedy pixel within 2e-2 of its maximum.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _net(seed=0):
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    torch.manual_seed(seed)
    return make_torch_qnet(6)


# ------------------------------------------------------------------------------------------------ CPU
def test_adam_state_round_trips_through_torch():
    """torch Adam stepped twice -> flat (params, m, v, step) -> torch format -> a fresh Adam loads it and its next step matches exactly"""
    from mujoco_rl_ur5_b200.qnet_learn import adam_from_torch, adam_to_torch

    net = _net(3)
    opt = torch.optim.Adam(net.parameters(), lr=0.002, betas=(0.8, 0.99), eps=1e-7, weight_decay=3e-5)
    g = torch.Generator().manual_seed(4)
    grads = [[torch.randn(p.shape, generator=g) * 0.01 for p in net.parameters()] for _ in range(3)]
    for step in range(2):
        for p, gr in zip(net.parameters(), grads[step]):
            p.grad = gr.clone()
        opt.step()
    m, v, step, hyper = adam_from_torch(opt.state_dict())
    assert step == 2 and hyper == dict(lr=0.002, betas=(0.8, 0.99), eps=1e-7, weight_decay=3e-5)
    names = [k for k, _ in net.named_parameters()]
    for k, p in net.named_parameters():
        assert torch.equal(m[k], opt.state[p]["exp_avg"]) and torch.equal(v[k], opt.state[p]["exp_avg_sq"])
    params = {k: p.detach().clone() for k, p in net.named_parameters()}
    sd = adam_to_torch(params, m, v, step, **hyper)
    net2 = _net(5)
    net2.load_state_dict(net.state_dict())
    opt2 = torch.optim.Adam(net2.parameters())
    opt2.load_state_dict(sd)
    for (p, p2), gr in zip(zip(net.parameters(), net2.parameters()), grads[2]):
        p.grad, p2.grad = gr.clone(), gr.clone()
    opt.step()
    opt2.step()
    for k, p, p2 in zip(names, net.parameters(), net2.parameters()):
        assert torch.equal(p, p2), k
    # no steps yet: no per-parameter state, as torch leaves a fresh optimiser
    assert adam_to_torch(params, m, v, 0, **hyper)["state"] == {}


def test_model_keys_are_the_reference_modules():
    from mujoco_rl_ur5_b200.qnet_learn import model_keys

    sd = _net(0).state_dict()
    assert model_keys() == list(sd.keys()) and len(sd) == 87
    assert sum("running" in k or "num_batches" in k for k in sd) == 36


def test_running_batchnorm_needs_running_statistics():
    from mujoco_rl_ur5_b200.qnet import QNetForward

    params = {k: v for k, v in _net(0).state_dict().items() if "running" not in k and "num_batches" not in k}
    with pytest.raises(ValueError):
        QNetForward(params, 0, batchnorm="running")
    with pytest.raises(ValueError):
        QNetForward(_net(0).state_dict(), 0, batchnorm="eval")


def test_dual_source_k_loop_barrier_protocol():
    """the k-step counts of the BN-folded blocks (9 taps x Ca/64 + Cx/64: 9*2+1, 9*1+2, 9*4+2, 9*8+4, 9*2+4) under the mbarrier model check
    of tests/host/pipeline_protocol_check.py (the second source changes which map the producer loads, not the ring protocol)"""
    sys.path.insert(0, os.path.join(HERE, "host"))
    import pipeline_protocol_check as pc

    n = 0
    for stages in (6, 8):
        for nk in (19, 11, 38, 76, 22):
            for ntiles in (1, 3, 5):
                pc.simulate(hash((stages, nk, ntiles)) & 0xffffffff, stages, nk, ntiles)
                n += 1
    assert n == 30


# ------------------------------------------------------------------------------------------------ GPU
def _stepped_net(seed=0, steps=3):
    """the fp32 torch module after a few seeded training-mode forwards: non-trivial running statistics"""
    net = _net(seed)
    g = torch.Generator().manual_seed(seed + 100)
    net.train()
    with torch.no_grad():
        for _ in range(steps):
            net(torch.rand((2, 4, 200, 200), generator=g))
    return net.eval()


@gpu
def test_bn_running_update_matches_float64():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    L = QNetLearner(seed=0)
    g = torch.Generator(device="cuda").manual_seed(3)
    B, HW, C = 5, 2500, 256
    x = torch.randn((B, HW, C), generator=g, device="cuda") * 1.7 + 0.4
    stats = torch.stack([x.sum(1), (x * x).sum(1)], dim=2).contiguous()
    L._merge(stats, B, C)
    rm = torch.rand(C, generator=g, device="cuda")
    rv = torch.rand(C, generator=g, device="cuda") + 0.5
    rm0, rv0 = rm.double(), rv.double()
    L._ck(L.L.gq_bn_running_update(L._p(stats), L._p(rm), L._p(rv), B, HW, C, 0.1, L._st()), "gq_bn_running_update")
    s = stats[0].double()
    mean = s[:, 0] / HW
    var = s[:, 1] / HW - mean * mean
    n = B * HW
    em, ev = 0.9 * rm0 + 0.1 * mean, 0.9 * rv0 + 0.1 * var * n / (n - 1)
    assert float(((rm.double() - em).abs() / em.abs().clamp_min(1e-3)).max()) <= 1e-6
    assert float(((rv.double() - ev).abs() / ev.abs()).max()) <= 1e-6


@gpu
def test_learner_running_statistics_match_torch_train_forward():
    """one learn_step on a batch of test_qnet_learn at each B = 3 (the golden batch), 1, 12 (the reference's BATCH_SIZE) and 15 (the offline
    trainer's): the 36 buffers against torch's train()-mode forward of the fp32 net on the same batch; relative error no worse than
    1.1 x what torch's own autocast-bf16 forward makes + 0.01"""
    for B in (3, 1, 12, 15):
        _check_running_statistics(B)


def _check_running_statistics(B):
    sys.path.insert(0, HERE)
    from test_qnet_learn import _batch, rel

    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    state, action, reward = _batch(B)
    net = _net(0)
    L = QNetLearner(net.state_dict(), 0)
    L.learn_step(state, action, reward)
    ours = L.model_state_dict()
    net32, net16 = _net(0).cuda().train(), _net(0).cuda().train()
    with torch.no_grad():
        net32(state.cuda())
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            net16(state.cuda())
    sd32, sd16 = net32.state_dict(), net16.state_dict()
    for k in sd32:
        if "running" in k:
            e, a = rel(ours[k], sd32[k].cpu()), rel(sd16[k].cpu(), sd32[k].cpu())
            assert e <= 1.1 * a + 0.01, (B, k, e, a)
        elif "num_batches" in k:
            assert int(ours[k]) == int(sd32[k]) == 1 and ours[k].dtype == torch.int64, (B, k)


def _ref_conv(a, w, bias, ks, relu, x=None, w3=None):
    y = F.conv2d(a.float(), w.float(), bias, padding=ks // 2)
    if x is not None:
        y = y + F.conv2d(x.float(), w3.float())
    return torch.relu(y) if relu else y


@gpu
@pytest.mark.parametrize("B,H,W,ca,cx,cout,relu", [(2, 50, 47, 128, 0, 64, True), (1, 50, 47, 64, 0, 256, False), (2, 50, 47, 128, 64, 128, True),
                                                    (3, 50, 50, 256, 512, 256, True), (2, 37, 41, 64, 128, 64, False), (1, 100, 100, 128, 64, 128, True)])
def test_conv_tc_fused_matches_torch(B, H, W, ca, cx, cout, relu):
    """gq_conv_tc_fused, single and dual source, both BLOCK_N instantiations, Ca != Cx, H*W not a multiple of 128"""
    from mujoco_rl_ur5_b200.qnet import QNetForward

    f = QNetForward(_net(0).state_dict(), 0)
    g = torch.Generator(device="cuda").manual_seed(B * 31 + ca + cx)
    a = torch.randn((B, ca, H, W), generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn((cout, ca, 3, 3), generator=g, device="cuda") / np.sqrt(9 * ca)).to(torch.bfloat16)
    bias = torch.randn(cout, generator=g, device="cuda")
    x = w3 = None
    wk = w.permute(0, 2, 3, 1).reshape(cout, 9 * ca)
    if cx:
        x = torch.randn((B, cx, H, W), generator=g, device="cuda").to(torch.bfloat16)
        w3 = (torch.randn((cout, cx, 1, 1), generator=g, device="cuda") / np.sqrt(cx)).to(torch.bfloat16)
        wk = torch.cat([wk, w3.reshape(cout, cx)], dim=1)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    ref = _ref_conv(a, w, bias, 3, relu, x, w3).permute(0, 2, 3, 1).reshape(B, H * W, cout)
    torch.backends.cudnn.allow_tf32 = tf32
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
    got = f.conv_tc_fused(nhwc(a), None if x is None else nhwc(x), wk.contiguous(), bias, B, H, W, ca, cx, cout, 3, relu).float()
    torch.cuda.synchronize()
    assert float((got - ref).abs().max()) <= 2 ** -8 * float(ref.abs().max()) + 2e-3  # bf16 output rounding + summation order


@gpu
def test_eval_forward_matches_fp32_eval_network():
    """whole network in eval mode against make_torch_qnet(6).eval() in fp32 with non-trivial running statistics, and batch / chunk
    independence: 7 images at once == 7 single-image forwards == max_batch=3, bit for bit"""
    from mujoco_rl_ur5_b200.qnet import QNetForward

    net = _stepped_net(0)
    sd = net.state_dict()
    assert float(sd["0.RB2.bn1.running_var"].sub(1).abs().max()) > 1e-3  # the statistics are not torch's initial ones
    state = torch.rand((7, 4, 200, 200), generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        ref = net(state)
    f = QNetForward(sd, 0, max_batch=64, batchnorm="running")
    n0 = f.launches
    q = f.forward(state.cuda())
    torch.cuda.synchronize()
    assert f.launches - n0 == 1 + 2 + 6 * 2 + 1 + 1  # first conv, 2 pools, 2 launches per BasicBlock, up-sampling, head
    err = (q.cpu() - ref).abs()
    assert float(err.mean()) <= 5e-3 and float(err.max()) <= 5e-2, (float(err.mean()), float(err.max()))
    act, val = f.greedy(q)
    flat = ref.reshape(7, -1)
    for i in range(7):
        j = int(act[i, 1]) * 40000 + int(act[i, 0])
        assert float(flat[i].max() - flat[i, j]) <= 2e-2
    singles = torch.cat([f.forward(state[i:i + 1].cuda()) for i in range(7)])
    assert torch.equal(q, singles)
    f3 = QNetForward(sd, 0, max_batch=3, batchnorm="running")
    assert torch.equal(q, f3.forward(state.cuda()))
    # the default keeps training-mode BatchNorm with per-image statistics
    fb = QNetForward(sd, 0)
    assert not torch.equal(fb.forward(state[:1].cuda()), q[:1])


@gpu
def test_checkpoints_round_trip_with_torch():
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    sys.path.insert(0, HERE)
    from test_qnet_learn import _golden_batch

    state, action, reward = _golden_batch()
    L = QNetLearner(seed=0)
    for _ in range(2):
        L.learn_step(state, action, reward)
    ck = L.checkpoint()
    net = make_torch_qnet(6)
    net.load_state_dict(ck["model_state_dict"], strict=True)
    assert list(ck["model_state_dict"]) == list(net.state_dict())
    assert all(v.device.type == "cpu" for v in ck["model_state_dict"].values())
    opt = torch.optim.Adam(net.parameters())
    opt.load_state_dict(ck["optimizer_state_dict"])
    assert opt.param_groups[0]["lr"] == L.lr and opt.param_groups[0]["weight_decay"] == L.wd
    # the same gradient: torch's next Adam step and gq_adam agree
    net = net.cuda()
    opt = torch.optim.Adam(net.parameters())
    opt.load_state_dict(ck["optimizer_state_dict"])
    g = torch.Generator(device="cuda").manual_seed(1)
    L.grad.copy_(torch.randn(L.grad.shape, generator=g, device="cuda") * 1e-3)
    for k, p in net.named_parameters():
        p.grad = L.g[k].clone()
    opt.step()
    L.step_count += 1
    L._ck(L.L.gq_adam(L._p(L.flat), L._p(L.grad), L._p(L.m), L._p(L.v), L.flat.numel(), L.lr, L.betas[0], L.betas[1], L.eps, L.wd, L.step_count,
                      L._st()), "gq_adam")
    for k, p in net.named_parameters():
        assert float((L.p[k] - p.detach()).abs().max()) <= 1e-6, k
    # a torch-written checkpoint restores everything, step count included
    ck_t = {"model_state_dict": {k: v.cpu() for k, v in net.state_dict().items()}, "optimizer_state_dict": opt.state_dict()}
    L2 = QNetLearner.from_checkpoint(ck_t, 0)
    assert L2.step_count == 3
    for k, p in net.named_parameters():
        st = opt.state[p]
        assert torch.equal(L2.p[k], p.detach()) and torch.equal(L2._flat_views(L2.m)[k], st["exp_avg"]) and torch.equal(L2._flat_views(L2.v)[k], st["exp_avg_sq"])
    back = L2.model_state_dict()
    for k, v in net.state_dict().items():
        assert torch.equal(back[k], v.cpu()), k
    # the eval forward of the learner is the running-statistics forward of its current state
    fw = L2.eval_forward(max_batch=2)
    assert fw.batchnorm == "running"
    q = fw.forward(state.cuda())
    assert q.shape == (3, 6, 200, 200) and bool(torch.isfinite(q).all())
