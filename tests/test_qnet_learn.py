"""Learner (SURVEY 8f.2): Grasp_Agent.learn() on the device — csrc/qnet_learn.cuh + mujoco_rl_ur5_b200/qnet_learn.py.

Reference: Grasping_Agent_multidiscrete.py:388-446 (gather-BCE loss, backward, Adam(lr, weight_decay 2e-5) :153-156).
Oracles: (1) tests/golden/qnet_learn_golden.json, one learn() step of the UNMODIFIED Modules.MULTIDISCRETE_RESNET on CPU in fp32
(make_learn_golden.py): loss, q_pred and per-parameter gradient checksums; (2) torch autograd in fp32 on the same tensors for every
backward building block and for every gradient tensor of the whole network (`qnet.make_torch_qnet` is pinned to the reference module by
the forward golden).  The kernels compute in bf16 with fp32 accumulation, so tolerances are relative L2 errors of a few 1e-3 per
building block (inputs pre-rounded to bf16) and a few 1e-2 for whole-network gradients.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qnet_learn_golden.json")


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _golden_batch(B=3):
    g = torch.Generator().manual_seed(5)
    state = torch.rand((B, 4, 200, 200), generator=g)
    action = torch.tensor([[3 * 40000 + 123 * 200 + 77], [0 * 40000 + 20 * 200 + 150], [5 * 40000 + 199 * 200 + 199]])
    reward = torch.tensor([[1.0], [0.0], [1.0]])
    return state, action, reward


def _batch(B):
    """the golden batch at B = 3; otherwise B seeded torch.rand states, random actions and alternating rewards 1, 0"""
    if B == 3:
        return _golden_batch()
    g = torch.Generator().manual_seed(50 + B)
    state = torch.rand((B, 4, 200, 200), generator=g)
    action = torch.randint(0, 6 * 200 * 200, (B, 1), generator=g)
    reward = (torch.arange(B) % 2 == 0).float().reshape(B, 1)
    return state, action, reward


def test_library_exports_the_learner_entry_points():
    import ctypes

    from mujoco_rl_ur5_b200.qnet import QLIB_PATH
    from mujoco_rl_ur5_b200.qnet_learn import LEARN_SYMBOLS

    lib = ctypes.CDLL(QLIB_PATH)
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "grasp_qnet.h")).read()
    for s in LEARN_SYMBOLS:
        assert hasattr(lib, s) and (s + "(") in header, s


def test_learner_refuses_to_run_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    with pytest.raises(RuntimeError):
        QNetLearner()


def test_torch_reference_reproduces_the_reference_repos_learn_step():
    """CPU: make_torch_qnet + autograd + torch Adam == the golden of the unmodified reference module (loss, q_pred, gradient and parameter checksums)"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    g = json.load(open(GOLD))
    torch.manual_seed(0)
    net = make_torch_qnet(6)
    opt = torch.optim.Adam(net.parameters(), lr=g["lr"], weight_decay=g["weight_decay"])
    state, action, reward = _golden_batch()
    q_pred = net(state).view(3, -1).gather(1, action)
    loss = F.binary_cross_entropy(q_pred, reward)
    loss.backward()
    assert abs(float(loss) - g["loss"]) < 1e-5
    assert np.abs(q_pred.detach().reshape(-1).numpy() - np.array(g["q_pred"])).max() < 1e-5
    for k, p in net.named_parameters():
        s, a = float(p.grad.double().sum()), float(p.grad.double().abs().sum())
        assert abs(a - g["grads"][k][1]) <= 2e-3 * g["grads"][k][1] + 1e-9, k
        assert abs(s - g["grads"][k][0]) <= 2e-3 * g["grads"][k][1] + 1e-9, k
    opt.step()
    for k, p in net.named_parameters():
        assert abs(float(p.detach().double().abs().sum()) - g["params_after_adam_step"][k][1]) <= 1e-4 * g["params_after_adam_step"][k][1] + 1e-6, k


# ------------------------------------------------------------------------------------------------ GPU: building blocks
@pytest.fixture(scope="module")
def learner():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    return QNetLearner(seed=0)


def _bf(x):
    return x.to(torch.bfloat16)


def _conv_case(B, ks, cin, cout, H, W):
    return pytest.param(B, ks, cin, cout, H, W, id=f"{ks}-{cin}-{cout}-{H}-{W}" + ("" if B == 3 else f"-B{B}"))  # (B = 3: the original ids)


@gpu
@pytest.mark.parametrize("B,ks,cin,cout,H,W", [_conv_case(3, 3, 64, 128, 20, 24), _conv_case(3, 1, 128, 64, 17, 9), _conv_case(3, 3, 128, 256, 10, 10),
                                               _conv_case(3, 3, 64, 64, 25, 25), _conv_case(3, 3, 256, 128, 30, 7), _conv_case(3, 1, 512, 256, 16, 16),
                                               _conv_case(1, 3, 64, 128, 20, 24), _conv_case(15, 1, 128, 64, 17, 9),
                                               # the learner's own convolutions at B = 12 (the reference's BATCH_SIZE) and 15 (the offline
                                               # trainer's): 100 x 100 and 50 x 50 maps end in a partial 128-pixel k-step
                                               _conv_case(12, 3, 64, 128, 100, 100), _conv_case(15, 3, 128, 256, 50, 50), _conv_case(12, 3, 256, 512, 50, 50),
                                               _conv_case(15, 1, 512, 256, 50, 50), _conv_case(15, 3, 128, 64, 100, 100)])
@pytest.mark.parametrize("nan_prefill", [1, 0])
def test_wgrad_and_dgrad_match_autograd(learner, B, ks, cin, cout, H, W, nan_prefill):
    """the wgmma weight-gradient kernel and the dgrad through the forward convolution.  Reference: autograd of F.conv2d in float64 on
    the same bf16 values.  The weight gradient's scratch and output buffers are, before the call:
    nan_prefill = 1: NaN, so that every split-K partial and every element of dW must be written by the call;
    nan_prefill = 0: the result of an identical earlier call, which the new result must equal bit for bit (partials summed in fixed order)"""
    g = torch.Generator(device="cuda").manual_seed(1)
    x = _bf(torch.randn((B, H, W, cin), generator=g, device="cuda"))
    dY = _bf(torch.randn((B, H, W, cout), generator=g, device="cuda"))
    w = (0.05 * torch.randn((cout, cin, ks, ks), generator=g, device="cuda"))
    wb = _bf(w)
    xr = x.double().permute(0, 3, 1, 2).clone().requires_grad_(True)
    wr = wb.double().clone().requires_grad_(True)
    y = F.conv2d(xr, wr, padding=ks // 2)
    y.backward(dY.double().permute(0, 3, 1, 2))
    # wgrad
    part = torch.empty(B * cout * ks * ks * cin, dtype=torch.float32, device="cuda")
    dW = torch.empty((cout, ks * ks, cin), dtype=torch.float32, device="cuda")

    def wgrad():
        learner._ck(learner.L.gq_conv_wgrad(learner._p(dY), learner._p(x), learner._p(part), learner._p(dW), B, H, W, cin, cout, ks, learner._st()), "gq_conv_wgrad")

    if nan_prefill:
        part.fill_(float("nan"))
        dW.fill_(float("nan"))
    else:
        wgrad()
        first = dW.clone()
    wgrad()
    if not nan_prefill:
        assert torch.equal(dW, first)
    e_w = rel(dW.view(cout, ks, ks, cin).permute(0, 3, 1, 2), wr.grad)
    # dgrad through the forward convolution kernel with flipped / transposed weights
    wT = wb.float().flip(2, 3).permute(1, 2, 3, 0).contiguous().to(torch.bfloat16)
    dx = learner._dgrad(dY.reshape(B, H * W, cout), wT.reshape(cin, ks * ks, cout), B, H, W, cin, cout, ks)
    e_x = rel(dx.view(B, H, W, cin).permute(0, 3, 1, 2), xr.grad)
    print(f"\nwgrad {e_w:.2e}  dgrad {e_x:.2e}")
    # fp32 accumulation of bf16 products (H100 80GB HBM3, 700 W: at most 1.1e-5 for wgrad, at 100 x 100 and B = 12 / 15, and 4.9e-6 for dgrad)
    assert e_w < 3e-5 and e_x < 3e-5, (e_w, e_x)


@gpu
@pytest.mark.parametrize("H,W", [(20, 24), (50, 47)])
def test_first_conv_wgrad_matches_autograd(learner, H, W):
    """gq_conv_first_wgrad (4 -> 64 channels, f32 NCHW input) against autograd of F.conv2d on the same values"""
    B = 3
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((B, 4, H, W), generator=g, device="cuda")
    dY = _bf(torch.randn((B, H, W, 64), generator=g, device="cuda"))
    wr = torch.zeros((64, 4, 3, 3), device="cuda", requires_grad=True)
    F.conv2d(x, wr, padding=1).backward(dY.float().permute(0, 3, 1, 2))
    n = B * H * W
    part = torch.empty(((n + 2047) // 2048) * 64 * 36, dtype=torch.float32, device="cuda")
    dW = torch.empty((64, 9, 4), dtype=torch.float32, device="cuda")
    learner._ck(learner.L.gq_conv_first_wgrad(learner._p(dY), learner._p(x), learner._p(part), learner._p(dW), B, H, W, learner._st()), "gq_conv_first_wgrad")
    assert rel(dW.view(64, 3, 3, 4).permute(0, 3, 1, 2), wr.grad) < 1e-3  # fp32 sums over B*H*W products in a different order (r02i: 2e-4 at 3 x 50 x 47)


@gpu
def test_bn_relu_backward_matches_autograd(learner):
    B, HW, Cc = 3, 500, 128
    g = torch.Generator(device="cuda").manual_seed(2)
    o = torch.randn((B, HW, Cc), generator=g, device="cuda") * 2 + 0.3
    gamma = torch.rand(Cc, generator=g, device="cuda") + 0.5
    beta = torch.randn(Cc, generator=g, device="cuda") * 0.1
    ident = torch.randn((B, HW, Cc), generator=g, device="cuda")
    dY = _bf(torch.randn((B, HW, Cc), generator=g, device="cuda"))
    orf = o.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    x4 = orf.permute(0, 2, 1).reshape(B, Cc, HW, 1)
    y = F.relu(F.batch_norm(x4, None, None, gr, br, training=True, eps=1e-5) + ident.permute(0, 2, 1).reshape(B, Cc, HW, 1))
    act = _bf(y.detach().reshape(B, Cc, HW).permute(0, 2, 1).contiguous())
    y.backward(dY.float().permute(0, 2, 1).reshape(B, Cc, HW, 1))
    # per-image (sum, sum of squares) as the convolution epilogue would write them, then merged over the batch
    stats = torch.stack([o.sum(1), (o * o).sum(1)], dim=2).contiguous()
    learner._merge(stats, B, Cc)
    d_o = torch.empty((B, HW, Cc), dtype=torch.bfloat16, device="cuda")
    dpre = torch.empty_like(d_o)
    part = torch.empty(((B * HW + 127) // 128) * Cc * 2, dtype=torch.float32, device="cuda")
    sums = torch.empty(2 * Cc, dtype=torch.float32, device="cuda")
    dg, db = torch.empty(Cc, device="cuda"), torch.empty(Cc, device="cuda")
    learner._ck(learner.L.gq_bn_relu_bwd(learner._p(dY), learner._p(act), learner._p(o), learner._p(stats), learner._p(gamma), B, HW, Cc, 1e-5, learner._p(dpre),
                                         learner._p(part), learner._p(sums), learner._p(dg), learner._p(db), learner._p(d_o), learner._st()), "gq_bn_relu_bwd")
    assert rel(d_o.float(), orf.grad) < 6e-3          # bf16 output
    assert rel(dg, gr.grad) < 1e-4 and rel(db, br.grad) < 1e-4
    assert rel(dpre.float(), dY.float() * (act.float() > 0)) == 0.0
    # the kernels move 8 channels per thread: other channel counts are refused
    o12 = torch.zeros((B, HW, 12), device="cuda")
    y12, d12 = torch.zeros((B, HW, 12), dtype=torch.bfloat16, device="cuda"), torch.empty((B, HW, 12), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="gq_bn_relu_bwd: C must be a multiple of 8"):
        learner._ck(learner.L.gq_bn_relu_bwd(learner._p(y12), learner._p(y12), learner._p(o12), learner._p(stats), learner._p(gamma), B, HW, 12, 1e-5, None,
                                             learner._p(part), learner._p(sums), None, None, learner._p(d12), learner._st()), "gq_bn_relu_bwd")


@gpu
def test_pool_upsample_backward_match_autograd(learner):
    B, H, W, Cc = 2, 21, 14, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    x = _bf(torch.randn((B, H, W, Cc), generator=g, device="cuda"))
    xr = x.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    y = F.max_pool2d(xr, 3, 2, 1)
    OH, OW = y.shape[2], y.shape[3]
    dY = _bf(torch.randn((B, OH, OW, Cc), generator=g, device="cuda"))
    y.backward(dY.float().permute(0, 3, 1, 2))
    dX = torch.empty((B, H, W, Cc), dtype=torch.bfloat16, device="cuda")
    learner._ck(learner.L.gq_maxpool_bwd(learner._p(x), learner._p(dY), learner._p(dX), B, H, W, Cc, learner._st()), "gq_maxpool_bwd")
    assert rel(dX.float().permute(0, 3, 1, 2), xr.grad) < 4e-3
    # 8 channels per thread: other channel counts are refused
    x12, dY12 = torch.zeros((B, H, W, 12), dtype=torch.bfloat16, device="cuda"), torch.zeros((B, OH, OW, 12), dtype=torch.bfloat16, device="cuda")
    dX12 = torch.empty((B, H, W, 12), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="gq_maxpool_bwd: C must be a multiple of 8"):
        learner._ck(learner.L.gq_maxpool_bwd(learner._p(x12), learner._p(dY12), learner._p(dX12), B, H, W, 12, learner._st()), "gq_maxpool_bwd")
    # bilinear x2, align_corners=True
    zr = torch.randn((B, Cc, H, W), generator=g, device="cuda").requires_grad_(True)
    up = F.interpolate(zr, scale_factor=2, mode="bilinear", align_corners=True)
    dU = _bf(torch.randn((B, 2 * H, 2 * W, Cc), generator=g, device="cuda"))
    up.backward(dU.float().permute(0, 3, 1, 2))
    dZ = torch.empty((B, H, W, Cc), dtype=torch.bfloat16, device="cuda")
    learner._ck(learner.L.gq_upsample2x_bwd(learner._p(dU), learner._p(dZ), B, H, W, Cc, learner._st()), "gq_upsample2x_bwd")
    assert rel(dZ.float().permute(0, 3, 1, 2), zr.grad) < 4e-3


@gpu
@pytest.mark.parametrize("saturate", [False, True])
def test_loss_head_backward_matches_float64(learner, saturate):
    """gq_loss_head_bwd at B = 12 on a [B,100,100,64] bf16 head input, with q from gq_head_up2 on that input, against float64 autograd of
    BCE(sigmoid(C1(UP2(x)))[action], r) in the reference's order (Modules.py:281-283, Grasping_Agent_multidiscrete.py:433-437).  Actions:
    the four corners, the four edges, odd and even interior coordinates (fractional bilinear weights; coincident taps merged at the last
    row / column), all six rotations, rewards 0 and 1.
    saturate=True: head biases +60 on rotation 0 and -120 on rotation 1 make q exactly 1.0 (with r = 0) and 0.0 (with r = 1) in fp32.
    There the spec is torch's fp32 chain (BCE backward divides by max(q(1-q), 1e-12), the sigmoid multiplies by q(1-q) = 0): loss 100,
    gradient 0.  float64 is no spec for such rows: it does not saturate between logits of about 16.6 and 37."""
    B, H, W, A = 12, 100, 100, 6
    fw = learner.fw
    g = torch.Generator(device="cuda").manual_seed(6)
    x = _bf(torch.rand((B, H, W, 64), generator=g, device="cuda") * 2)  # non-negative, as the ReLU output it stands for
    w_head, b_head = fw.w_head, fw.b_head.clone()
    if saturate:
        b_head[0] += 60.0
        b_head[1] -= 120.0
    yx = [(0, 0), (199, 0), (0, 199), (199, 199), (0, 77), (120, 199), (199, 64), (33, 0), (123, 77), (50, 150), (101, 98), (2, 181)]
    rot = torch.arange(B) % 6
    action = torch.tensor([int(r) * 40000 + y * 200 + xx for r, (y, xx) in zip(rot, yx)], device="cuda")
    reward = torch.tensor([0, 1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1], dtype=torch.float32, device="cuda")  # rotation 0: r = 0 twice, rotation 1: r = 1 twice
    sat = (rot < 2).cuda() if saturate else torch.zeros(B, dtype=torch.bool, device="cuda")
    z = torch.empty((B, A, H, W), device="cuda")
    q = torch.empty((B, A, 2 * H, 2 * W), device="cuda")
    learner._ck(learner.L.gq_head_up2(learner._p(x), learner._p(w_head), learner._p(b_head), learner._p(z), learner._p(q), B, H, W, A, learner._st()), "gq_head_up2")
    loss_terms, qsel = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    dX = torch.empty((B, H * W, 64), dtype=torch.bfloat16, device="cuda")
    dWp, dbp = torch.empty((B, A, 64), device="cuda"), torch.empty((B, A), device="cuda")
    dW, db = torch.empty((A, 64), device="cuda"), torch.empty(A, device="cuda")
    learner._ck(learner.L.gq_loss_head_bwd(learner._p(q), learner._p(x), learner._p(w_head), learner._p(action), learner._p(reward), B, A, H, W, learner._p(loss_terms),
                                           learner._p(qsel), learner._p(dX), learner._p(dWp), learner._p(dbp), learner._p(dW), learner._p(db), learner._st()),
                "gq_loss_head_bwd")
    torch.cuda.synchronize()
    assert torch.equal(qsel, q.reshape(B, -1).gather(1, action[:, None])[:, 0])
    # float64 reference
    xr = x.double().permute(0, 3, 1, 2).clone().requires_grad_(True)
    wr = w_head.double().reshape(A, 64, 1, 1).clone().requires_grad_(True)
    br = b_head.double().clone().requires_grad_(True)
    v = F.conv2d(F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=True), wr, br).reshape(B, -1).gather(1, action[:, None])[:, 0]
    terms = F.binary_cross_entropy(torch.sigmoid(v), reward.double(), reduction="none")
    # saturated rows enter with torch fp32's gradient (checked just below: 0), i.e. without one
    (torch.where(sat, terms.detach(), terms).sum() / B).backward()
    if saturate:
        assert bool((qsel[sat] == (rot[sat.cpu()] == 0).float().cuda()).all()), qsel  # q exactly 1.0 / 0.0 in fp32
        v32 = v.detach().float()[sat].clone().requires_grad_(True)
        t32 = F.binary_cross_entropy(torch.sigmoid(v32), reward[sat], reduction="none")
        (t32.sum() / B).backward()
        assert bool((t32 == 100.0).all()) and bool((v32.grad == 0).all()), (t32, v32.grad)
        assert bool((loss_terms[sat] == 100.0).all()), loss_terms
        assert not bool(dX[sat].any()) and not bool(dW[:2].any()) and not bool(db[:2].any()), (dW[:2].abs().max(), db[:2])
    err = {"loss_terms": rel(loss_terms, terms.detach()), "dX": rel(dX.view(B, H, W, 64).permute(0, 3, 1, 2), xr.grad),
           "dW": rel(dW, wr.grad.reshape(A, 64)), "db": rel(db, br.grad)}
    print("\nloss/head backward (saturate=%s): " % saturate + "  ".join(f"{k} {e:.2e}" for k, e in err.items()))
    # H100 80GB HBM3 (700 W), both cases: loss_terms 3.4e-7 (q from the fp32 head, C1 before UP2), dX 1.7e-3 (bf16), dW 1.5e-6, db 2.1e-7
    bound = {"loss_terms": 1e-6, "dX": 4e-3, "dW": 4e-6, "db": 6e-7}
    bad = {k: (e, bound[k]) for k, e in err.items() if not e <= bound[k]}
    assert not bad, bad


@gpu
def test_adam_step_matches_torch(learner):
    n = 10007
    g = torch.Generator(device="cuda").manual_seed(4)
    p = torch.randn(n, generator=g, device="cuda")
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=0.001, weight_decay=0.00002)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for step in (1, 2, 3):
        grad = torch.randn(n, generator=g, device="cuda") * 0.01
        ref.grad = grad.clone()
        opt.step()
        learner._ck(learner.L.gq_adam(learner._p(p), learner._p(grad), learner._p(m), learner._p(v), n, 0.001, 0.9, 0.999, 1e-8, 0.00002, step, learner._st()), "gq_adam")
        assert (p - ref.detach()).abs().max() < 1e-6  # one fp32 unit in the last place at |p| ~ 4


# ------------------------------------------------------------------------------------------------ GPU: the whole step
@gpu
def test_learn_step_matches_the_reference(learner):
    """one learn() step at each batch size B = 3 (the golden batch), 1, 12 (the reference's BATCH_SIZE) and 15 (the offline trainer's):
    at B = 3, loss / q_pred against the reference repo's numbers (golden); at every B, the training-mode Q-map against torch's fp32 train()
    forward over the same batch, EVERY gradient tensor against torch autograd of the pinned fp32 network, parameters after Adam against
    torch.optim.Adam where the gradient is not rounding noise"""
    for B in (3, 1, 12, 15):
        _check_learn_step(B)


def _check_learn_step(B):
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    gold = json.load(open(GOLD))
    state, action, reward = _batch(B)
    torch.manual_seed(0)
    net = make_torch_qnet(6)
    L = QNetLearner(net.state_dict(), 0, lr=gold["lr"], weight_decay=gold["weight_decay"])
    net = net.cuda().train()
    opt = torch.optim.Adam(net.parameters(), lr=gold["lr"], weight_decay=gold["weight_decay"])
    qmap = net(state.cuda())
    q_pred = qmap.view(B, -1).gather(1, action.cuda())
    loss_ref = F.binary_cross_entropy(q_pred, reward.cuda())
    loss_ref.backward()
    q, saved = L.forward_train(state)
    # the whole Q-map, BatchNorm over the batch: the bars of test_qnet.py's per-image forward against the fp32 network
    err = (q - qmap.detach().reshape(q.shape)).abs()
    print("B=%d Q-map: mean |err| %.2e, max %.2e" % (B, float(err.mean()), float(err.max())))
    assert float(err.mean()) <= 5e-3 and float(err.max()) <= 5e-2, (B, float(err.mean()), float(err.max()))
    loss, qsel = L.backward(q, saved, action, reward)
    if B == 3:
        assert abs(float(loss) - gold["loss"]) < 2e-2 and np.abs(qsel.cpu().numpy() - np.array(gold["q_pred"])).max() < 2e-2
    worst = {}
    for k, p in net.named_parameters():
        worst[k] = rel(L.g[k], p.grad)
    # what bf16 activations cost torch itself: the same network under autocast(bfloat16) against its own fp32 gradients.  The loss
    # gradient enters at ONE pixel per image, so the backward signal is carried by few units and a handful of ReLU masks that differ
    # between the bf16 and the fp32 forward move the early layers' gradients by tens of per cent - for torch exactly as for these kernels.
    net16 = make_torch_qnet(6)
    net16.load_state_dict({k: v for k, v in net.state_dict().items()})
    net16 = net16.cuda().train()
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        q16 = net16(state.cuda()).float().view(B, -1).gather(1, action.cuda())
    F.binary_cross_entropy(q16, reward.cuda()).backward()
    auto = {k: rel(p16.grad, p.grad) for (k, p16), (_, p) in zip(net16.named_parameters(), net.named_parameters())}
    for k in worst:
        print("  %-24s ours vs fp32 %.4f   torch-autocast-bf16 vs fp32 %.4f" % (k, worst[k], auto[k]))
    print("learn step B=%d: loss %.5f (fp32 torch %.5f), worst gradient relative L2 error %.4f (%s)" % (B, float(loss), float(loss_ref), max(worst.values()),
                                                                                                       max(worst, key=worst.get)))
    # The bar is torch's OWN bf16 path (autocast) against the same fp32 gradients: the loss touches 3 of 120 000 head
    # outputs, so a bf16 rounding that flips a ReLU mask upstream moves an early-layer gradient by tens of per cent in
    # either bf16 implementation (measured r02f: ours 0.30..0.46, autocast 0.36..0.60 in the first trunk; the head
    # conv 0.050 vs 0.058, its bias 0.009 vs 0.018).  Every layer must be no worse than 1.1x autocast's error + 1 %.
    assert worst["1.C1.bias"] < 0.03, (B, worst["1.C1.bias"])
    assert worst["1.C1.weight"] < 0.10, (B, worst["1.C1.weight"])
    bad = {k: (v, auto[k]) for k, v in worst.items() if v > 1.1 * auto[k] + 0.01}
    assert not bad, (B, bad)
    # gradient checksums of the reference repo itself on the golden batch (abs-sum is robust to bf16 rounding)
    for k in (gold["grads"] if B == 3 else ()):
        a = float(L.g[k].double().abs().sum())
        tol = 0.05 if k.startswith("1.C1") else 0.6  # (see above: early layers carry the bf16-vs-fp32 mask noise)
        assert abs(a - gold["grads"][k][1]) <= tol * gold["grads"][k][1] + 1e-8, (k, a, gold["grads"][k][1])
    # optimiser: same update as torch.optim.Adam given the SAME gradient (our own), and close to the reference's step where |g| is well above noise
    ref_params = {k: p.detach().clone() for k, p in net.named_parameters()}
    opt.step()
    before = {k: v.clone() for k, v in L.p.items()}
    L.step_count += 1
    L._ck(L.L.gq_adam(L._p(L.flat), L._p(L.grad), L._p(L.m), L._p(L.v), L.flat.numel(), L.lr, 0.9, 0.999, 1e-8, L.wd, 1, L._st()), "gq_adam")
    for k, p in net.named_parameters():
        big = p.grad.abs() > 20 * p.grad.abs().mean() * 0.05 + 1e-7
        upd_ref = (p.detach() - ref_params[k])[big]
        upd = (L.p[k] - before[k])[big]
        if upd_ref.numel():
            agree = (torch.sign(upd) == torch.sign(upd_ref)).float().mean()
            assert agree > (0.97 if k.startswith("1.C1") else 0.75), (k, float(agree))  # early layers: the mask noise above
            # first Adam step: |update| = lr * |g| / (|g| + eps), i.e. lr wherever OUR gradient is not ~1e-8; `big` is chosen on the fp32
            # reference gradient, so a bf16-noise-cancelled element can slip in (r02j: one element at 0.8 lr): all but 0.1 % within 10 %
            assert ((upd.abs() - 0.001).abs() < 1e-4).float().mean() > 0.999, k


@gpu
def test_two_learn_steps_reduce_the_loss_on_a_fixed_batch():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    state, action, reward = _golden_batch()
    L = QNetLearner(seed=0, lr=0.001)
    losses = [L.learn_step(state, action, reward) for _ in range(4)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


def test_gradient_groups_partition_the_parameters():
    """the per-group all-reduce of the multi-GPU learner covers every parameter exactly once, each group contiguous in the flat buffer"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    names = [k for k, v in make_torch_qnet(6).state_dict().items() if v.dtype.is_floating_point and "running" not in k]
    seen = []
    for pre in QNetLearner.GROUPS:
        idx = [i for i, k in enumerate(names) if k.startswith(pre)]
        assert idx and idx == list(range(idx[0], idx[-1] + 1)), pre
        seen += idx
    assert sorted(seen) == list(range(len(names)))
