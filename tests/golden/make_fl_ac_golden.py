#!/usr/bin/env python
"""fl_ac_golden.npz: the REFERENCE's actor aggregation (Envs/PathPlan_City.py:590-601, Federated_Learning_AC) executed here on
real reference SAC trainers.

The method is called unbound on a minimal stand-in whose .Agents[i].Trainer are reference SAC_Trainers (continuous branch, the
shipped shape: actor 100-64-{2, 2}, critics 102-64-64-2).  The trainers are named fl_ac_<g>, so SAC_Trainer.__init__ finds no
checkpoint under the reference's Mod/ (the name UAV_0 would load the shipped Mod/*_SAC_UAV_0.pth).

What the reference computes: global = deepcopy(actor_0); global.state_dict()[k] += actor_i.state_dict()[k] for i = 1 .. G-1
(state_dict tensors share storage with the parameters, so the sum lands in `global`); then
global.state_dict()[k] = torch.div(...) assigns into a temporary dict and is lost; finally replace_param(global) copies global
into every trainer's actor.  Every actor therefore becomes the float32 sum theta_0 + ... + theta_{G-1}, not the mean.  This
script asserts that, and that the critics, the target critics, every optimiser state and log_alpha are untouched.

Recorded: G, the actors before (actor0, [G][P]) and after (actor1, [G][P]), in state_dict order (fc1, fc_mu, fc_std).  To keep
the fixture small the initial parameters lie on a grid of multiples of 2^-13 inside the torch.nn.Linear init range.
Run in the build container only:  python tests/golden/make_fl_ac_golden.py"""
import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness  # noqa: E402

ref_harness.load_reference()
import torch  # noqa: E402
import Envs.PathPlan_City as ppc  # noqa: E402  (reference)
from FactoryClass.TrainerFactory import TrainerFactory  # noqa: E402  (reference)

G, OBS, H, A = 5, 100, 64, 2


def flat(net):
    return np.concatenate([p.detach().numpy().ravel() for p in net.state_dict().values()]).astype(np.float32)


def load_flat(net, vec):
    off = 0
    with torch.no_grad():
        for p in net.state_dict().values():
            n = p.numel()
            p.copy_(torch.from_numpy(vec[off:off + n].reshape(p.shape)))
            off += n
    assert off == vec.size


class _Agent:
    def __init__(self, tr):
        self.Trainer = tr


class _Env:
    def __init__(self, agents):
        self.Agents = agents


def sac_param(g):
    return {"Trainer_Type": "SAC_Trainer", "Is_Train": "1", "IsPriority_Replay": "0", "name": "fl_ac_%d" % g,
            "actor": {"NetWork": "PolicyNetContinuous_SAC", "h": "1", "w": str(OBS), "channel": "1", "action_bound": "1",
                      "hiden_dim": str(H), "output": str(A), "lr": "0.0001"},
            "critic": {"NetWork": "QValueNetContinuous_SAC", "h": "1", "w": str(OBS), "channel": "1", "hiden_dim": str(H),
                       "action_dim": str(A), "lr": "0.001"},
            "SAC_param": {"IS_Continuous": "1", "alpha_lr": "0.0001", "target_entropy": "1", "gamma": "0.99", "tau": "0.05"},
            "replay_size": "10000", "LEARNING_RATE": "0.0005", "Batch_Size": "64", "max_epoch": "100",
            "save_loop": "1000000000"}


def grid_actor(rng):
    """One flat actor vector (fc1 [H][OBS], fc1.b, fc_mu [A][H], fc_mu.b, fc_std [A][H], fc_std.b), every block
    U(+-1/sqrt(fan_in)) like torch.nn.Linear's init, on multiples of 2^-13."""
    parts = []
    for r, c in ((H, OBS), (A, H), (A, H)):
        m = int(8192 / np.sqrt(c))
        parts += [rng.integers(-m, m + 1, size=r * c), rng.integers(-m, m + 1, size=r)]
    return (np.concatenate(parts) * 2.0 ** -13).astype(np.float32)


def others(tr):
    """Everything Federated_Learning_AC must leave alone: critics, targets, the three optimisers, log_alpha and its optimiser."""
    nets = [flat(getattr(tr, nm)) for nm in ("critic_1", "critic_2", "target_critic_1", "target_critic_2")]
    opts = [copy.deepcopy(getattr(tr, nm).state_dict()) for nm in
            ("actor_optimizer", "critic_1_optimizer", "critic_2_optimizer", "log_alpha_optimizer")]
    return nets, opts, float(tr.log_alpha.item())


def same_opt(a, b):
    if a.keys() != b.keys() or a["param_groups"] != b["param_groups"] or a["state"].keys() != b["state"].keys():
        return False
    return all(torch.equal(a["state"][i][k], b["state"][i][k]) for i in a["state"] for k in a["state"][i])


def main():
    rng = np.random.default_rng(23)
    trainers = []
    for g in range(G):
        torch.manual_seed(300 + g)
        tr = TrainerFactory().Create_Trainer(sac_param(g))
        assert tr is not None and tr.epoch == 0, "a checkpoint was loaded"
        trainers.append(tr)
    actor0 = np.stack([grid_actor(rng) for _ in range(G)])
    for t, v in zip(trainers, actor0):
        load_flat(t.actor, v)
    # one optimiser step on the critics and alpha so their states are not empty when checked
    for t in trainers:
        for opt, net in ((t.critic_1_optimizer, t.critic_1), (t.critic_2_optimizer, t.critic_2)):
            opt.zero_grad()
            sum(p.sum() for p in net.parameters()).backward()
            opt.step()
    before = [others(t) for t in trainers]
    ppc.PathPlan_City.Federated_Learning_AC(_Env([_Agent(t) for t in trainers]))
    actor1 = np.stack([flat(t.actor) for t in trainers])
    for t, (nets, opts, la) in zip(trainers, before):
        nets2, opts2, la2 = others(t)
        assert all(np.array_equal(x, y) for x, y in zip(nets, nets2)), "critics / targets must be left untouched"
        assert all(same_opt(x, y) for x, y in zip(opts, opts2)), "optimiser states must be left untouched"
        assert la == la2, "log_alpha must be left untouched"
    # every actor is the left-to-right float32 sum, not the mean
    s = actor0[0].copy()
    for g in range(1, G):
        s = (s + actor0[g]).astype(np.float32)
    assert all(np.array_equal(a, s) for a in actor1), "every actor must be the sum of all actors"
    assert not np.array_equal(actor1[0], (s / np.float32(G)).astype(np.float32))
    res = {"G": np.int64(G), "actor0": actor0, "actor1": actor1, "torch_version": np.array(torch.__version__)}
    np.savez_compressed(os.path.join(HERE, "fl_ac_golden.npz"), **res)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in res.items()})


if __name__ == "__main__":
    main()
