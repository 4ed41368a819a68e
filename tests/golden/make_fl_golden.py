#!/usr/bin/env python
"""fl_golden.npz: the REFERENCE's selective federated aggregation (Envs/PathPlan_City.py:644-684,
Federated_Learning_choice) executed here on real reference trainers.

The method is called unbound on a minimal stand-in whose .Agents[i].Trainer are reference trainers (DDQN_Trainer with
QValueNet_SAC, DuelingDQN_Trainer with VAnet2; obs 100, 27 actions).  DDQN_Trainer has no replace_param, so its
instances get DuelingDQN_Trainer's (a parameter copy into q_local).  Each trainer's replay_memory.memory is filled
with Transition tuples directly and random.sample is patched to a recorded tape, so the probe states are known.  The
module's `sorted` is wrapped to record every round's chosen list.  Recorded per case: q_local of every trainer before
and after, the probe states of every round, the chosen trainers of every round (q_target is checked here to stay as it
was and is not recorded).

To keep the fixture small the networks are 100-16(-16)-27 and the initial parameters and probe states lie on a grid of
multiples of 2^-13 inside the torch.nn.Linear init range (they compress to about 1.5 bytes each); the parameters after
aggregation carry full float32 mantissas.

Cases:
  ddqn5    G = 5 DDQN trainers, independent initialisations.  The generator asserts that a Jacobi restatement (every
           loss and every average from the initial parameters) gives different parameters: the case discriminates the
           in-place round order.
  duel6    G = 6 Dueling trainers.  Trainer 1 is trainer 0 plus small noise, trainers 4 and 5 are bit-identical (trainer
           0 plus larger noise): round 0 ranks 4 and 5 with exactly equal losses at the boundary of the kept half, and
           the stable sort keeps the lower index.
Run in the build container only:  python tests/golden/make_fl_golden.py"""
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ref_harness  # noqa: E402

ref_harness.load_reference()
import torch  # noqa: E402
import Envs.PathPlan_City as ppc  # noqa: E402  (reference)
from FactoryClass.TrainerFactory import TrainerFactory  # noqa: E402  (reference)
from Trainer.DuelingDQN_Trainer import DuelingDQN_Trainer  # noqa: E402  (reference)
import fl_restatement as flr  # noqa: E402

S, NA, OBS, H = 10, 27, 100, 16


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


def run_case(name, trainer_type, net, G, rng, tweak=None):
    trainers = []
    for g in range(G):
        torch.manual_seed(100 + g)
        param = {"Trainer_Type": trainer_type, "NetWork": net, "w": str(OBS), "hiden_dim": str(H),
                 "output": str(NA), "name": "fl_%s_%d" % (name, g), "LEARNING_RATE": "0.0005",
                 "Batch_Size": "64", "gamma": "0.99", "save_loop": "1000000000",
                 "replay_size": "10000", "Update_loop": "3", "Is_Train": "1"}
        tr = TrainerFactory().Create_Trainer(param)
        if not hasattr(tr, "replace_param"):
            # only DuelingDQN_Trainer defines replace_param (DuelingDQN_Trainer.py:204-207); DDQN_Trainer gets the same method
            tr.replace_param = types.MethodType(DuelingDQN_Trainer.replace_param, tr)
        trainers.append(tr)
    hidden, dueling = ([H, H], False) if net == "QValueNet_SAC" else ([H], True)
    local0 = np.stack([grid_params(rng, hidden, dueling) for _ in range(G)])
    if tweak is not None:
        tweak(local0, rng)
    for t, v in zip(trainers, local0):
        load_flat(t.q_local, v)
    target0 = np.stack([flat(t.q_target) for t in trainers])
    # replay contents: 40 transitions per trainer, states in the env's observation range
    n_mem = 40
    mem_states = (rng.integers(-8192, 8193, size=(G, n_mem, OBS)) * 2.0 ** -13).astype(np.float32)
    for g, t in enumerate(trainers):
        t.replay_memory.memory = [(torch.tensor(mem_states[g, i:i + 1]), torch.tensor([[0]]), torch.tensor([[0.0]]),
                                   torch.tensor(mem_states[g, i:i + 1]), torch.tensor([[0.0]])) for i in range(n_mem)]
    tape = np.stack([rng.choice(n_mem, size=S, replace=False) for _ in range(G)]).astype(np.int64)
    probes = np.stack([mem_states[g, tape[g]] for g in range(G)])
    calls = [0]
    chosen = []
    orig_sample, orig_sorted = random.sample, ppc.__dict__.get("sorted", sorted)

    def sample_tape(population, k):
        g = calls[0]
        calls[0] += 1
        assert k == S
        return [population[int(i)] for i in tape[g]]

    def sorted_rec(seq, key=None, reverse=False):
        out = orig_sorted(seq, key=key, reverse=reverse)
        chosen.append([int(it[0]) for it in out[:len(out) // 2]])
        return out

    random.sample = sample_tape
    ppc.sorted = sorted_rec
    try:
        ppc.PathPlan_City.Federated_Learning_choice(_Env([_Agent(t) for t in trainers]))
    finally:
        random.sample = orig_sample
        del ppc.sorted
    assert calls[0] == G and len(chosen) == G
    local1 = np.stack([flat(t.q_local) for t in trainers])
    target1 = np.stack([flat(t.q_target) for t in trainers])
    assert np.array_equal(target0, target1), "q_target must be left untouched"
    k = (G - 1) // 2
    ch = np.full((G, max(1, k)), -1, np.int64)
    for p, c in enumerate(chosen):
        ch[p, :len(c)] = c
    # the in-order restatement reproduces the reference; a Jacobi restatement does not
    mine, my_chosen, _ = flr.federate(local0, probes, OBS, hidden, NA, dueling)
    assert np.array_equal(my_chosen, ch), (my_chosen, ch)
    assert np.array_equal(mine, local1)
    jac, _, _ = flr.federate(local0, probes, OBS, hidden, NA, dueling, jacobi=True)
    assert not np.array_equal(jac, local1), "case does not discriminate the round order"
    return {"local0": local0, "local1": local1, "probes": probes, "tape": tape, "chosen": ch,
            "G": np.int64(G), "dueling": np.int64(dueling), "hidden": np.asarray(hidden, np.int64)}


def grid_params(rng, hidden, dueling):
    """One flat parameter vector: every block U(+-1/sqrt(fan_in)) like torch.nn.Linear's init, on multiples of 2^-13."""
    parts = []
    for r, c in flr.layers(OBS, hidden, NA, dueling):
        m = int(8192 / np.sqrt(c))
        parts += [rng.integers(-m, m + 1, size=r * c), rng.integers(-m, m + 1, size=r)]
    return (np.concatenate(parts) * 2.0 ** -13).astype(np.float32)


def tie_tweak(local0, rng):
    base = local0[0].copy()
    local0[1] = base + (rng.integers(-8, 9, size=base.shape) * 2.0 ** -13).astype(np.float32)
    twin = base + (rng.integers(-160, 161, size=base.shape) * 2.0 ** -13).astype(np.float32)
    local0[4] = twin
    local0[5] = twin


if __name__ == "__main__":
    rng = np.random.default_rng(11)
    res = {}
    for name, tt, net, G, tw in (("ddqn5", "DDQN_Trainer", "QValueNet_SAC", 5, None),
                                 ("duel6", "DuelingDQN_Trainer", "VAnet2", 6, tie_tweak)):
        for k, v in run_case(name, tt, net, G, rng, tw).items():
            res["%s_%s" % (name, k)] = v
    assert res["duel6_chosen"][0].tolist() == [1, 4], res["duel6_chosen"][0]
    res["cases"] = np.array(["ddqn5", "duel6"])
    res["torch_version"] = np.array(torch.__version__)
    np.savez_compressed(os.path.join(HERE, "fl_golden.npz"), **res)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in res.items()})
