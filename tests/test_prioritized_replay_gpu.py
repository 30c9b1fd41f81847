"""Prioritized experience replay on the GPU: the sum-tree kernels and the stratified sampler against the numpy mirror of
tests/test_prioritized_replay.py, the importance-weighted loss and learn step against float64 / fp32 torch autograd, and the trainer
with `prioritized` on (determinism, the priorities it writes back, checkpoints, the CLI)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_prioritized_replay import TreeMirror, build_tree, sample_mirror

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALPHA, EPS = 0.6, 1e-6


def _replay(size, alpha=ALPHA, eps=EPS):
    from mujoco_rl_ur5_b200.replay_buffer import PrioritizedObservationReplay

    return PrioritizedObservationReplay(size, (2, 2), device="cuda", alpha=alpha, eps=eps)


def _push(rp, k, n):
    """n fake 2x2 transitions numbered k, k+1, ... (the tree only sees the slots they claim)"""
    rgb = torch.zeros((n, 2, 2, 3), dtype=torch.uint8, device="cuda")
    depth = torch.arange(k, k + n, dtype=torch.float32, device="cuda")[:, None, None].expand(n, 2, 2).contiguous()
    rp.push_batch(rgb, depth, torch.arange(k, k + n), torch.zeros(n), torch.arange(k, k + n), torch.zeros(n, dtype=torch.int64))


def _within_ulp(a, b, n=4):
    return bool(np.all(np.abs(a - b) <= n * np.spacing(np.abs(b))))


def _check_tree(rp, m, where):
    tree = rp.tree.cpu().numpy()
    k = np.arange(1, rp.cap)
    assert np.array_equal(tree[k], tree[2 * k] + tree[2 * k + 1]), where  # every internal node = the exact f64 sum of its children
    # leaves: CUDA's double pow is not correctly rounded (glibc's is), so within 4 ulp rather than bit for bit
    assert _within_ulp(tree[rp.cap:], m.leaves()), (where, np.abs(tree[rp.cap:] - m.leaves()).max())
    assert _within_ulp(np.array([float(rp.pmax)]), np.array([m.pmax])), (where, float(rp.pmax), m.pmax)
    return tree


@pytest.mark.parametrize("size", [2000, 16385])
def test_tree_follows_pushes_and_updates(size):
    rp, m = _replay(size), TreeMirror(size)
    assert rp.cap == m.cap
    rng = np.random.RandomState(size)
    k = 0

    def push(n):
        nonlocal k
        _push(rp, k, n)
        m.push([j % size for j in range(k + max(0, n - size), k + n)])  # transition j lives in slot j % size; of a push > size the last size survive
        k += n

    def update(B, raise_pmax=False):
        idx = rng.randint(0, len(rp), B)
        if B >= 8:  # duplicates inside the batch: the last one's priority stays
            idx[B // 2:B // 2 + 3] = idx[1]
            idx[-1] = idx[0]
        q = rng.rand(B).astype(np.float32)
        r = (rng.rand(B) < 0.3).astype(np.float32)
        if raise_pmax:  # |r - q| > 1 (not a sigmoid output, but the kernel does not care): priorities above 1 raise pmax
            q[2] = -0.75
            r[2] = 1.0
        rp.update_priorities(torch.from_numpy(idx).cuda(), torch.from_numpy(q).cuda(), torch.from_numpy(r).cuda())
        m.update(idx, q, r, ALPHA, EPS)

    ops = [lambda: push(700), lambda: update(12), lambda: push(size // 2 + 3), lambda: update(64), lambda: push(size - 5),  # wrap-around
           lambda: update(12, True), lambda: push(size + 37),                                                             # larger than the ring
           lambda: update(1), lambda: update(12), lambda: push(1), lambda: update(1024, True), lambda: push(4096)]
    for i, op in enumerate(ops):
        op()
        _check_tree(rp, m, (size, i))
    assert m.pmax > 1.0 and len(rp) == size


def _filled_tree(size, length, seed):
    rp, m = _replay(size), TreeMirror(size)
    _push(rp, 0, length)
    m.push(np.arange(length))
    rng = np.random.RandomState(seed)
    for _ in range(5):
        idx = rng.randint(0, length, 200)
        q = rng.rand(200).astype(np.float32)
        r = (rng.rand(200) < 0.2).astype(np.float32)
        rp.update_priorities(torch.from_numpy(idx).cuda(), torch.from_numpy(q).cuda(), torch.from_numpy(r).cuda())
        m.update(idx, q, r, ALPHA, EPS)
    return rp


@pytest.mark.parametrize("size,length", [(2000, 2000), (2000, 1234), (16385, 9000)])
def test_sampling_equals_the_mirror(size, length):
    rp = _filled_tree(size, length, size + length)
    tree = rp.tree.cpu().numpy()
    for B in (1, 12, 64):
        for seed, update, rank, beta in ((0, 0, 0, 0.4), (77, 12345, 0, 0.4), (77, 12345, 1, 0.7), (2 ** 40 + 3, 2 ** 33 + 9, 7, 1.0)):
            idx, w = rp.sample_slots(B, beta, seed, update, rank)
            w_idx, w_w = sample_mirror(tree, rp.cap, length, B, beta, seed, update, rank)
            key = (B, seed, update, rank)
            assert np.array_equal(idx.cpu().numpy(), w_idx), key
            got = w.cpu().numpy().astype(np.float64)
            want = w_w.astype(np.float32).astype(np.float64)  # computed in double, stored as f32
            assert np.all(np.abs(got - want) <= 1e-12 * want), (key, got, want)
            assert (w_idx < length).all() and (tree[rp.cap + w_idx] > 0).all()


def test_sampling_edges_on_hand_built_trees():
    """all mass in slot 0 (an empty right subtree at every level), u at the total (the last strata of a 1024 batch), empty left subtrees"""
    for leaves, length in (([2.5] + [0.0] * 15, 1), ([0.1, 0.2, 0.3, 0.0, 0.0], 3), ([0.0, 0.0, 0.0, 0.0, 1.0, 1e-300], 6)):
        rp = _replay(len(leaves))
        m = build_tree(leaves)
        rp.tree.copy_(torch.from_numpy(m.tree))
        rp.length = length
        for B in (1, 64, 1024):
            for update in range(3):
                idx, _ = rp.sample_slots(B, 0.4, 5, update, 0)
                idx = idx.cpu().numpy()
                assert np.array_equal(idx, sample_mirror(m.tree, m.cap, length, B, 0.4, 5, update, 0)[0])
                assert (m.tree[m.cap + idx] > 0).all(), (leaves, B)


def test_sampled_frequencies_follow_the_priorities():
    from scipy.stats import chisquare

    size = 300  # cap 512: the leaves past 300 stay empty
    rp = _replay(size, alpha=1.0, eps=0.0)  # p = |r - q|: the priorities are set directly
    _push(rp, 0, size)
    i = np.arange(size)
    p = (0.05 + 2.0 * (i % 10 == 0) + 0.5 * (i % 7 == 3) + i / 300.0).astype(np.float32)
    rp.update_priorities(torch.from_numpy(i).cuda(), torch.from_numpy(p).cuda(), torch.zeros(size, device="cuda"))
    B, n_upd = 100, 1000
    draws = torch.cat([rp.sample_slots(B, 0.4, 31, u, 0)[0] for u in range(n_upd)]).cpu().numpy()
    counts = np.bincount(draws, minlength=rp.cap)
    assert counts[size:].sum() == 0
    expect = B * n_upd * p.astype(np.float64) / p.astype(np.float64).sum()
    # stratification spreads each batch over the whole mass, so the counts vary less than multinomial ones: the statistic sits below
    # its degrees of freedom, and a wrong proportion (a slot off by a few per cent) still pushes it far above them
    stat, pval = chisquare(counts[:size], expect)
    print(f"\nchi2 {stat:.1f} over {size - 1} dof, p = {pval:.3f}")
    assert pval > 1e-3, (stat, pval)


# ------------------------------------------------------------------------------------------------ weighted loss and learner
@pytest.fixture(scope="module")
def learner():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    return QNetLearner(seed=0)


def _bf(x):
    return x.to(torch.bfloat16)


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _head_call(learner, fn, q, x, action, reward, weight, B, A, H, W):
    loss_terms, qsel = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    dX = torch.empty((B, H * W, 64), dtype=torch.bfloat16, device="cuda")
    dWp, dbp = torch.empty((B, A, 64), device="cuda"), torch.empty((B, A), device="cuda")
    dW, db = torch.empty((A, 64), device="cuda"), torch.empty(A, device="cuda")
    p = learner._p
    w = () if weight is None else (p(weight),)
    learner._ck(getattr(learner.L, fn)(p(q), p(x), p(learner.fw.w_head), p(action), p(reward), *w, B, A, H, W, p(loss_terms), p(qsel), p(dX), p(dWp),
                                       p(dbp), p(dW), p(db), learner._st()), fn)
    torch.cuda.synchronize()
    return dict(loss_terms=loss_terms, qsel=qsel, dX=dX, dW=dW, db=db)


@pytest.mark.parametrize("saturate", [False, True])
def test_weighted_loss_head_backward_matches_float64(learner, saturate):
    """gq_loss_head_bwd_weighted against float64 autograd of binary_cross_entropy(q, r, weight=w), in the setting and with the bars of
    tests/test_qnet_learn.py::test_loss_head_backward_matches_float64 (saturated rows: torch fp32's loss 100 and zero gradient); with
    w = 1 its outputs equal gq_loss_head_bwd's bit for bit"""
    B, H, W, A = 12, 100, 100, 6
    fw = learner.fw
    g = torch.Generator(device="cuda").manual_seed(6)
    x = _bf(torch.rand((B, H, W, 64), generator=g, device="cuda") * 2)
    b_head = fw.b_head.clone()
    if saturate:
        b_head[0] += 60.0
        b_head[1] -= 120.0
    yx = [(0, 0), (199, 0), (0, 199), (199, 199), (0, 77), (120, 199), (199, 64), (33, 0), (123, 77), (50, 150), (101, 98), (2, 181)]
    rot = torch.arange(B) % 6
    action = torch.tensor([int(r) * 40000 + y * 200 + xx for r, (y, xx) in zip(rot, yx)], device="cuda")
    reward = torch.tensor([0, 1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1], dtype=torch.float32, device="cuda")
    weight = (0.05 + 0.95 * torch.rand(B, generator=g, device="cuda")).float()
    weight[3] = 1.0  # the batch's largest weight, as gq_per_sample normalises
    sat = (rot < 2).cuda() if saturate else torch.zeros(B, dtype=torch.bool, device="cuda")
    z = torch.empty((B, A, H, W), device="cuda")
    q = torch.empty((B, A, 2 * H, 2 * W), device="cuda")
    learner._ck(learner.L.gq_head_up2(learner._p(x), learner._p(fw.w_head), learner._p(b_head), learner._p(z), learner._p(q), B, H, W, A, learner._st()), "gq_head_up2")
    out = _head_call(learner, "gq_loss_head_bwd_weighted", q, x, action, reward, weight, B, A, H, W)
    # w = 1: the unweighted kernel's bits
    ones = _head_call(learner, "gq_loss_head_bwd_weighted", q, x, action, reward, torch.ones(B, device="cuda"), B, A, H, W)
    plain = _head_call(learner, "gq_loss_head_bwd", q, x, action, reward, None, B, A, H, W)
    for k in plain:
        assert torch.equal(ones[k], plain[k]), k
    # float64 reference: F.binary_cross_entropy(q, r, weight=w) = mean(w * terms)
    xr = x.double().permute(0, 3, 1, 2).clone().requires_grad_(True)
    wr = fw.w_head.double().reshape(A, 64, 1, 1).clone().requires_grad_(True)
    br = b_head.double().clone().requires_grad_(True)
    v = F.conv2d(F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=True), wr, br).reshape(B, -1).gather(1, action[:, None])[:, 0]
    terms = F.binary_cross_entropy(torch.sigmoid(v), reward.double(), reduction="none")
    wd = weight.double()
    loss64 = (wd * torch.where(sat, terms.detach(), terms)).sum() / B
    if not saturate:
        assert abs(float(loss64) - float(F.binary_cross_entropy(torch.sigmoid(v), reward.double(), weight=wd))) < 1e-15
    loss64.backward()
    if saturate:
        assert bool((out["loss_terms"][sat] == 100.0 * weight[sat]).all()), out["loss_terms"]
        assert not bool(out["dX"][sat].any()) and not bool(out["dW"][:2].any()) and not bool(out["db"][:2].any())
    err = {"loss_terms": rel(out["loss_terms"], wd * terms.detach()), "dX": rel(out["dX"].view(B, H, W, 64).permute(0, 3, 1, 2), xr.grad),
           "dW": rel(out["dW"], wr.grad.reshape(A, 64)), "db": rel(out["db"], br.grad)}
    print("\nweighted loss/head backward (saturate=%s): " % saturate + "  ".join(f"{k} {e:.2e}" for k, e in err.items()))
    bound = {"loss_terms": 1e-6, "dX": 4e-3, "dW": 4e-6, "db": 6e-7}  # test_loss_head_backward_matches_float64's bars
    bad = {k: (e, bound[k]) for k, e in err.items() if not e <= bound[k]}
    assert not bad, bad


def _batch(B):
    g = torch.Generator().manual_seed(50 + B)
    state = torch.rand((B, 4, 200, 200), generator=g)
    action = torch.randint(0, 6 * 200 * 200, (B, 1), generator=g)
    reward = (torch.arange(B) % 2 == 0).float().reshape(B, 1)
    weight = (0.1 + 0.9 * torch.rand(B, generator=g)).float()
    weight[0] = 1.0
    return state, action, reward, weight


def test_weighted_learn_step_matches_torch():
    """learn_step(weight=w) at B = 12 against fp32 torch autograd of binary_cross_entropy(q_pred, r, weight=w): the whole-network bars of
    tests/test_qnet_learn.py (every gradient no worse than 1.1 x torch's own bf16 autocast error + 1 %, the head within 3 % / 10 %)"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    B = 12
    state, action, reward, weight = _batch(B)
    torch.manual_seed(0)
    net = make_torch_qnet(6)
    L = QNetLearner(net.state_dict(), 0)
    net = net.cuda().train()
    q_pred = net(state.cuda()).view(B, -1).gather(1, action.cuda())
    loss_ref = F.binary_cross_entropy(q_pred, reward.cuda(), weight=weight.cuda()[:, None])
    loss_ref.backward()
    loss, qsel = L.learn_step(state, action, reward, return_pred=True, weight=weight.cuda())
    assert abs(loss - float(loss_ref)) < 2e-2 * max(1.0, float(loss_ref)), (loss, float(loss_ref))
    assert float((qsel - q_pred.detach()[:, 0]).abs().max()) < 5e-2
    worst = {k: rel(L.g[k], p.grad) for k, p in net.named_parameters()}
    net16 = make_torch_qnet(6)
    net16.load_state_dict({k: v for k, v in net.state_dict().items()})
    net16 = net16.cuda().train()
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        q16 = net16(state.cuda()).float().view(B, -1).gather(1, action.cuda())
    F.binary_cross_entropy(q16, reward.cuda(), weight=weight.cuda()[:, None]).backward()
    auto = {k: rel(p16.grad, p.grad) for (k, p16), (_, p) in zip(net16.named_parameters(), net.named_parameters())}
    print("\nweighted learn step B=12: loss %.5f (fp32 torch %.5f), worst gradient %.4f (%s)" % (loss, float(loss_ref), max(worst.values()),
                                                                                                max(worst, key=worst.get)))
    assert worst["1.C1.bias"] < 0.03 and worst["1.C1.weight"] < 0.10, (worst["1.C1.bias"], worst["1.C1.weight"])
    bad = {k: (v, auto[k]) for k, v in worst.items() if v > 1.1 * auto[k] + 0.01}
    assert not bad, bad


def test_unit_weights_step_like_the_unweighted_learner():
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    state, action, reward, _ = _batch(12)
    torch.manual_seed(0)
    sd = make_torch_qnet(6).state_dict()
    a, b = QNetLearner(sd, 0), QNetLearner(sd, 0)
    for _ in range(2):
        la = a.learn_step(state, action, reward)
        lb = b.learn_step(state, action, reward, weight=torch.ones(12, device="cuda"))
        assert la == lb
    assert torch.equal(a.flat, b.flat) and torch.equal(a.m, b.m) and torch.equal(a.v, b.v)


# ------------------------------------------------------------------------------------------------ trainer
PER = dict(alpha=ALPHA, beta0=0.4, beta_updates=12, eps=EPS)


def _trainer(n, **kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    return BatchedTrainer(n, "A", 0, **kw)


def test_prioritized_training_is_deterministic_and_writes_the_priorities(tmp_path):
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.replay_buffer import PrioritizedObservationReplay

    paths = []
    for run in range(2):
        tr = _trainer(64, seed=11, updates_per_step=2, prioritized=PER)
        assert isinstance(tr.replay, PrioritizedObservationReplay)
        seen = []
        if run == 0:  # after each update, the sampled slots' leaves = (|r - qsel| + eps)^alpha of the returned qsel (later duplicate wins)
            orig = tr.replay.update_priorities

            def check(idx, qsel, reward):
                orig(idx, qsel, reward)
                i, q, r = idx.cpu().numpy(), qsel.cpu().numpy(), reward.reshape(-1).cpu().numpy()
                p = (np.abs(r.astype(np.float64) - q.astype(np.float64)) + EPS) ** ALPHA
                want = {int(s): v for s, v in zip(i, p)}
                leaves = tr.replay.tree[tr.replay.cap:].cpu().numpy()
                got = np.array([leaves[s] for s in want])
                assert _within_ulp(got, np.array(list(want.values()))), (got, want)
                assert (i < len(tr.replay)).all()
                seen.append(len(i))

            tr.replay.update_priorities = check
        try:
            tr.train(2, 3)
            assert tr.learner.step_count == 2 * 6
            if run == 0:
                assert seen == [12] * 12
            os.makedirs(str(tmp_path / f"run{run}"))
            p = str(tmp_path / f"run{run}" / "ck.pt")
            ck = tr.save(p)
            paths.append(p)
        finally:
            tr.close()
    assert open(paths[0], "rb").read() == open(paths[1], "rb").read()
    from tests.test_batched_train import REFERENCE_KEYS

    loaded = torch.load(paths[0], map_location="cpu", weights_only=False)
    assert set(loaded) == REFERENCE_KEYS and set(ck) == REFERENCE_KEYS
    net = make_torch_qnet(6)
    net.load_state_dict(loaded["model_state_dict"], strict=True)
    opt = torch.optim.Adam(net.parameters())
    opt.load_state_dict(loaded["optimizer_state_dict"])
    assert float(opt.state[next(iter(net.parameters()))]["step"]) == 12


def test_cli_trains_with_prioritized_replay(tmp_path):
    import json

    out = str(tmp_path / "w.pt")
    r = subprocess.run([sys.executable, "-m", "mujoco_rl_ur5_b200.batched_train", "--envs", "64", "--episodes", "1", "--steps-per-episode", "3",
                        "--updates-per-step", "2", "--prioritized", "--per-alpha", "0.7", "--per-beta0", "0.5", "--out", out], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    recs = [json.loads(ln) for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(recs) == 3 and all(rec["updates"] == 2 and np.isfinite(rec["mean_loss"]) for rec in recs)
    assert os.path.exists(out)
