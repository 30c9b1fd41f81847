"""Offline training of the grasp Q-network on recorded transitions: the reference's `Offline RL/train.py` on the device.

    trainer = OfflineTrainer("Data/..._total_of_6081_transitions.pt", device=0)   # files of offline_data / the reference's scripts
    history = trainer.run()                                                       # one dict of metrics per epoch
    trainer.save("weights.pt")                                                    # {"model_state_dict", "optimizer_state_dict"}

or `python -m mujoco_rl_ur5_b200.offline_train DATA.pt --epochs 20 --out weights.pt`.

What it computes, with line numbers of train.py:
* the whole data file stays on the device (u8 RGB + f32 depth; 6 081 transitions are 1.7 GB); each batch is gathered there and transformed
  by `QNetForward.obs_to_state_train` (depth clipped at 1.1, N(0, 0.001) noise, ColorJitter(0.5, 0.5, 0.5, 0.5); grasping_dataset.py:42-74).
  Both splits go through this transform, because the reference's Dataset applies it in __getitem__;
* training: one `QNetLearner.learn_step` per batch, the short last batch included (:102-124); evaluation of the test split after every
  epoch with the eval-mode forward (`QNetLearner.eval_forward`, BatchNorm with running statistics: `policy_net.eval()`, :167-195);
* metrics: `binary_accuracy` (:198-224, thresholds 0.5 / 0.3, 0 for a class absent from the batch) and `AverageMeter` (:227-252;
  losses weighted by batch size, accuracies by label counts).

Random numbers: the same torch stream as the reference.  `torch.manual_seed(seed)` (:28), `random_split` 80/20 (:69-71), the network's
construction (:76, also when a checkpoint is loaded afterwards), then per epoch the training DataLoader (shuffle=True) and the test one,
each drawing its iterator seed and its sampler seed from the default generator, and every sample drawing its ColorJitter parameters
(randperm(4) + 4 uniforms) in __getitem__.  torch's own DataLoader runs over an index dataset whose __getitem__ makes exactly those draws,
so the batch order and the jitter factors equal the reference's.  Only the depth noise differs: it comes from the counter-based device
generator keyed on (seed, transition index, epoch) instead of `np.random.normal`.  The colour arithmetic is torchvision's float-tensor
form of ColorJitter, where the reference jitters a PIL (uint8) image.
"""
import argparse
import time

import numpy as np

from . import offline_data
from .qnet import make_torch_qnet
from .qnet_learn import QNetLearner, check_optimizer

DEPTH_THRESHOLD = 1.1  # grasping_dataset.py:45
NOISE_STD = 0.001      # grasping_dataset.py:51
JITTER = 0.5           # ColorJitter(brightness=0.5, contrast=0.5, saturation=0.5, hue=0.5), grasping_dataset.py:21


def binary_accuracy(predictions, targets, positive_threshold=0.5, negative_threshold=0.3):
    """-> (positive accuracy, number of positive labels, negative accuracy, number of negative labels) of one batch.  A positive counts
    as correct when its prediction is above `positive_threshold`, a negative when below `negative_threshold`; the accuracy of a class
    with no label in the batch is 0."""
    import torch

    with torch.no_grad():
        p, t = predictions.reshape(-1), targets.reshape(-1)
        n_pos = t.sum().item()
        n_neg = t.numel() - n_pos
        pos_ok = ((p > positive_threshold) & (t == 1)).sum().item()
        neg_ok = ((p < negative_threshold) & (t == 0)).sum().item()
    return (pos_ok / n_pos if n_pos != 0 else 0), n_pos, (neg_ok / n_neg if n_neg != 0 else 0), n_neg


class AverageMeter:
    """running weighted mean: update(value, n) adds value with weight n; `avg` is 0 until a weight arrives"""

    def __init__(self, name=""):
        self.name = name
        self.reset()

    def reset(self):
        self.val, self.sum, self.count, self.avg = 0, 0, 0, 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        if self.count > 0:
            self.avg = self.sum / self.count


class _JitteredIndex:
    """dataset of transition indices whose __getitem__ draws the sample's ColorJitter parameters from the default torch generator, as
    torchvision's ColorJitter.get_params does inside the reference's Grasping_Dataset.__getitem__: (index, factors [4], order [4])"""

    def __init__(self, n, strength=JITTER):
        self.n, self.s = n, strength

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        import torch

        s = self.s
        order = torch.randperm(4)
        fac = [float(torch.empty(1).uniform_(max(0.0, 1 - s), 1 + s)) for _ in range(3)] + [float(torch.empty(1).uniform_(-s, s))]
        return i, torch.tensor(fac, dtype=torch.float32), order.to(torch.int32)


def rng_setup(n, batch_size=15, seed=30):
    """train.py's start in its order (:28, :69-76): -> (network, train loader, test loader).  Iterating a loader yields
    (indices [b] int64, jitter factors [b,4] f32, operation order [b,4] int32) per batch and draws what the reference draws."""
    import torch
    from torch.utils.data import DataLoader, random_split

    torch.manual_seed(seed)
    ds = _JitteredIndex(n)
    train_size = int(0.8 * n)
    trainset, testset = random_split(ds, [train_size, n - train_size])
    train_loader = DataLoader(dataset=trainset, batch_size=batch_size, shuffle=True)
    test_loader = DataLoader(dataset=testset, batch_size=batch_size, shuffle=True)
    net = make_torch_qnet(6)
    return net, train_loader, test_loader


def rng_plan(n, epochs, batch_size=15, seed=30):
    """the batches and jitter parameters of `epochs` epochs without training (training draws no random numbers):
    [{"train": [(indices, factors, order), ...], "test": [...]}, ...] as lists"""
    _, train_loader, test_loader = rng_setup(n, batch_size, seed)
    out = []
    for _ in range(epochs):
        out.append({k: [(i.tolist(), f.tolist(), o.tolist()) for i, f, o in loader] for k, loader in (("train", train_loader), ("test", test_loader))})
    return out


class OfflineTrainer:
    def __init__(self, data, device=0, batch_size=15, lr=1e-3, weight_decay=2e-5, epochs=20, seed=30, load=None, optimizer=None, momentum=0.9):
        """data: path of a transition file (offline_data / the reference's generate_data, unite_data, extract_positives) or the tuple
        offline_data.load_transitions returns; load: None, a checkpoint path or a {"model_state_dict", "optimizer_state_dict"} dict;
        optimizer: "adam" or "sgd" (torch.optim.SGD with `momentum`); None is Adam for a fresh run and the checkpoint's optimiser
        with `load`, which also brings its own lr, momentum and weight decay"""
        import torch

        check_optimizer("adam" if optimizer is None else optimizer, 1, momentum)
        opt = {} if optimizer is None else {"optimizer": optimizer}

        self.torch = torch
        self.dev = torch.device("cuda", device)
        rgb, depth, actions, rewards = offline_data.load_transitions(data) if isinstance(data, str) else data
        self.n = len(actions)
        if self.n < 2:
            raise ValueError("the data file needs at least two transitions")
        self.H, self.W = int(depth.shape[1]), int(depth.shape[2])
        self.batch_size, self.epochs, self.seed = int(batch_size), int(epochs), int(seed)
        net, self.train_loader, self.test_loader = rng_setup(self.n, self.batch_size, self.seed)
        if load is not None:
            ckpt = load if isinstance(load, dict) else torch.load(load, map_location="cpu", weights_only=False)
            self.learner = QNetLearner.from_checkpoint(ckpt, device, **opt)  # lr / weight decay from the checkpoint, as optimizer.load_state_dict does (:86)
        else:
            self.learner = QNetLearner(net.state_dict(), device, lr=lr, weight_decay=weight_decay, momentum=momentum, **opt)
        del net
        self.rgb = torch.as_tensor(np.ascontiguousarray(rgb)).to(self.dev)
        self.depth = torch.as_tensor(np.ascontiguousarray(depth, dtype=np.float32)).to(self.dev)
        self.actions = torch.as_tensor(np.asarray(actions, dtype=np.int64)).to(self.dev)
        self.rewards = torch.as_tensor(np.asarray(rewards, dtype=np.int64)).to(self.dev)
        self.epoch = 0
        self.history = []
        self.last_test = []  # (indices, factors, order, q_pred) of the latest evaluation, batch by batch

    def states(self, idx, factors, order, epoch):
        """the network inputs [b,4,H,W] f32 of transitions `idx` in `epoch`, gathered and transformed on the device"""
        t = self.torch
        i = idx.to(self.dev, t.int64)
        obs = {"rgb": self.rgb.index_select(0, i), "depth": self.depth.index_select(0, i)}
        return self.learner.fw.obs_to_state_train(obs, DEPTH_THRESHOLD, NOISE_STD, seed=self.seed, step=epoch, env_index=i,
                                                  jitter=factors.to(self.dev).contiguous(), order=order.to(self.dev, t.int32).contiguous())

    def train_epoch(self):
        self.epoch += 1
        loss_m, pos_m, neg_m = AverageMeter("Training Loss"), AverageMeter("Training positive Accuracy"), AverageMeter("Training negative Accuracy")
        for idx, fac, order in self.train_loader:
            i = idx.to(self.dev)
            state = self.states(idx, fac, order, self.epoch)
            reward = self.rewards.index_select(0, i)
            loss, q_pred = self.learner.learn_step(state, self.actions.index_select(0, i), reward, return_pred=True)
            loss_m.update(loss, len(idx))
            pa, npos, na, nneg = binary_accuracy(q_pred, reward)
            pos_m.update(pa, npos)
            neg_m.update(na, nneg)
        return loss_m.avg, pos_m.avg, neg_m.avg

    def evaluate(self):
        """the test split through the eval-mode forward (BatchNorm with running statistics), then gather and BCE"""
        t = self.torch
        F = t.nn.functional
        fw = self.learner.eval_forward()
        loss_m, pos_m, neg_m = AverageMeter("Test Loss"), AverageMeter("Test Positive Accuracy"), AverageMeter("Test Negative Accuracy")
        self.last_test = []
        with t.no_grad():
            for idx, fac, order in self.test_loader:
                i = idx.to(self.dev)
                q = fw.forward(self.states(idx, fac, order, self.epoch))
                q_pred = q.view(len(idx), -1).gather(1, self.actions.index_select(0, i).view(-1, 1))
                reward = self.rewards.index_select(0, i).view(-1, 1)
                loss_m.update(float(F.binary_cross_entropy(q_pred, reward.float())), len(idx))
                pa, npos, na, nneg = binary_accuracy(q_pred, reward)
                pos_m.update(pa, npos)
                neg_m.update(na, nneg)
                self.last_test.append((idx, fac, order, q_pred.view(-1).clone()))
        return loss_m.avg, pos_m.avg, neg_m.avg

    def run(self, epochs=None, log=None):
        """train for `epochs` (default: the constructor's) more epochs, evaluating after each; -> the history of every epoch so far"""
        for _ in range(self.epochs if epochs is None else int(epochs)):
            t0 = time.perf_counter()
            tr = self.train_epoch()
            te = self.evaluate()
            self.torch.cuda.synchronize(self.dev)
            rec = dict(epoch=self.epoch, train_loss=tr[0], train_pos_acc=tr[1], train_neg_acc=tr[2], test_loss=te[0], test_pos_acc=te[1],
                       test_neg_acc=te[2], seconds=time.perf_counter() - t0)
            self.history.append(rec)
            if log:
                log("epoch %(epoch)d: train loss %(train_loss).4f pos %(train_pos_acc).4f neg %(train_neg_acc).4f | test loss %(test_loss).4f "
                    "pos %(test_pos_acc).4f neg %(test_neg_acc).4f (%(seconds).1f s)" % rec)
        return self.history

    def checkpoint(self):
        return self.learner.checkpoint()

    def save(self, path):
        """writes {"model_state_dict", "optimizer_state_dict"} like train.py:147-163 (loads into Modules.MULTIDISCRETE_RESNET + Adam, or
        SGD with "learner_step" added)"""
        self.torch.save(self.checkpoint(), path)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Offline RL/train.py on the GPU: train the grasp Q-network on a transition file")
    ap.add_argument("data")
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=15)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--weight-decay", type=float, default=2e-5)
    ap.add_argument("--seed", type=int, default=30)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--load", default=None, help="checkpoint to continue from ({'model_state_dict', 'optimizer_state_dict'})")
    ap.add_argument("--out", default=None, help="where to save the final checkpoint")
    ap.add_argument("--optimizer", choices=("adam", "sgd"), default=None, help="adam, or sgd with momentum (default: the --load checkpoint's, else adam)")
    ap.add_argument("--momentum", type=float, default=0.9, help="SGD momentum of a fresh run (a loaded checkpoint keeps its own)")
    a = ap.parse_args(argv)
    try:
        check_optimizer(a.optimizer or "adam", 1, a.momentum)
    except ValueError as e:
        ap.error(str(e))
    tr = OfflineTrainer(a.data, a.device, a.batch_size, a.lr, a.weight_decay, a.epochs, a.seed, a.load, optimizer=a.optimizer, momentum=a.momentum)
    t0 = time.perf_counter()
    tr.run(log=print)
    dt = time.perf_counter() - t0
    print(f"training ({a.epochs} epochs, {tr.n} transitions) took {dt:.1f} s")
    if a.out:
        tr.save(a.out)
        print(f"saved network weights and optimizer state to {a.out}")


if __name__ == "__main__":
    main()
