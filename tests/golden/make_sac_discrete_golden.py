#!/usr/bin/env python
"""Generate tests/golden/sac_discrete_golden.npz by EXECUTING THE PYTHON REFERENCE.

Run in the build container only (needs the reference):   python tests/golden/make_sac_discrete_golden.py

SAC_Trainer with <IS_Continuous>0</IS_Continuous> and PolicyNet_SAC / QValueNet_SAC (Trainer/SAC_Trainer.py:380-430,
BaseClass/BaseCNN.py:296-343) at the shipped shape 100-64-27: three consecutive update(transition_dict) calls on synthetic
B = 64 batches with done rows and every action index present.

Kept small: the seeded initial parameters are rounded to multiples of 2^-10 (and the targets copied from the rounded critics,
as the reference's constructor copies them), the states are multiples of 1/64, and after each step the parameters and Adam
moments are recorded at a fixed stratified sample of NSAMPLE flat indices that covers every tensor (every fc3 bias whole).
Full per-step vectors of the five networks and their moments would take about 1.9 MB of incompressible floats.  Recorded:
  sacd_actor0, sacd_critic_10, sacd_critic_20   initial flat parameters (state_dict order); the targets equal the critics
  sacd_idx                    the sampled flat indices (the actor and the critics share one layout)
  sacd_s / a / r / s2 / d     the batches, [K][B][...]
  sacd_<net>                  parameters of actor, critic_1, critic_2, target_critic_1, target_critic_2 at sacd_idx after
                              each step, [K][NSAMPLE]
  sacd_<net>_m / _v           Adam exp_avg / exp_avg_sq of actor, critic_1, critic_2 at sacd_idx after each step, [K][NSAMPLE]
  sacd_log_alpha / _m / _v    log_alpha and its Adam moments after each step, [K]
  sacd_actor_loss, sacd_critic_1_loss, sacd_critic_2_loss   per step (the critic losses captured from F.mse_loss)
  sacd_probs                  actor(s) on each step's batch states before that step, [K][B][A]
  sacd_keys / sacd_shapes     the state_dict keys and shapes of the actor and the critic
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness  # noqa: E402

ref_harness.load_reference()              # chdir into oracle/_work, seeds everything with 42
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

NETS = ("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")
B, K, A, OBS, HID = 64, 3, 27, 100, 64
NSAMPLE = 1024


def sample_indices(rng, sizes):
    """a sorted stratified sample of flat indices: every tensor proportionally, at least 16 entries each, the last bias whole"""
    out, off = [], 0
    for i, n in enumerate(sizes):
        m = n if i == len(sizes) - 1 else min(n, max(16, round(NSAMPLE * n / sum(sizes))))
        out.append(off + np.sort(rng.choice(n, m, replace=False)))
        off += n
    return np.concatenate(out).astype(np.int32)


def flat(t_list):
    return np.concatenate([t.detach().numpy().ravel() for t in t_list]).astype(np.float32)


def synth(rng):
    s = (rng.integers(-64, 65, size=(B, OBS)) / 64.0).astype(np.float32)
    s2 = (rng.integers(-64, 65, size=(B, OBS)) / 64.0).astype(np.float32)
    a = np.concatenate([np.arange(A), rng.integers(0, A, B - A)]).astype(np.int32)
    rng.shuffle(a)
    r = rng.normal(-2.0, 6.0, size=B).astype(np.float32)
    d = (rng.uniform(size=B) < 0.15).astype(np.float32)
    d[:2] = 1.0
    return s, a, r, s2, d


def main():
    from FactoryClass.TrainerFactory import TrainerFactory
    rng = np.random.default_rng(23)
    torch.manual_seed(2718)
    param = {"Trainer_Type": "SAC_Trainer", "Is_Train": "1", "IsPriority_Replay": "0", "name": "golden_sacd",
             "actor": {"NetWork": "PolicyNet_SAC", "h": "1", "w": str(OBS), "channel": "1", "hiden_dim": str(HID),
                       "output": str(A), "lr": "0.0001"},
             "critic": {"NetWork": "QValueNet_SAC", "h": "1", "w": str(OBS), "channel": "1", "hiden_dim": str(HID),
                        "output": str(A), "lr": "0.001"},
             "SAC_param": {"IS_Continuous": "0", "alpha_lr": "0.0001", "target_entropy": "1", "gamma": "0.99", "tau": "0.05"},
             "replay_size": "10000", "LEARNING_RATE": "0.0005", "Batch_Size": str(B), "max_epoch": "100",
             "save_loop": "1000000000"}
    tr = TrainerFactory().Create_Trainer(param)
    assert tr is not None and tr.IS_Continuous == 0
    tr.replay_memory.memory = [0] * (B + 1)               # only its length gates training (:384)
    with torch.no_grad():                                  # round the seeded init in place (the optimisers hold these tensors)
        for nm in NETS[:3]:
            for p in getattr(tr, nm).parameters():
                p.copy_(torch.round(p * 1024.0) / 1024.0)
        tr.target_critic_1.load_state_dict(tr.critic_1.state_dict())
        tr.target_critic_2.load_state_dict(tr.critic_2.state_dict())
    out = {}
    for nm in NETS[:3]:
        out["sacd_%s0" % nm] = flat(getattr(tr, nm).state_dict().values())
    idx = sample_indices(rng, [v.numel() for v in tr.actor.state_dict().values()])
    assert [v.numel() for v in tr.actor.state_dict().values()] == [v.numel() for v in tr.critic_1.state_dict().values()]
    out["sacd_idx"] = idx
    out["sacd_log_alpha0"] = np.float32(tr.log_alpha.item())
    out["sacd_hparams"] = np.array([1e-4, 1e-3, 1e-4, 1.0, 0.99, 0.05], np.float64)  # actor_lr critic_lr alpha_lr target_entropy gamma tau
    out["sacd_keys"] = np.array([k for k in tr.actor.state_dict()] + [k for k in tr.critic_1.state_dict()])
    out["sacd_shapes"] = np.array([list(v.shape) + [0] * (2 - v.dim()) for v in tr.actor.state_dict().values()] +
                                  [list(v.shape) + [0] * (2 - v.dim()) for v in tr.critic_1.state_dict().values()], np.int64)
    mse_seen = []
    orig_mse = F.mse_loss

    def mse(x, y, *a, **k):
        v = orig_mse(x, y, *a, **k)
        mse_seen.append(float(v))
        return v
    F.mse_loss = mse
    rec = {k: [] for k in ("s", "a", "r", "s2", "d", "probs", "actor_loss", "critic_1_loss", "critic_2_loss",
                           "log_alpha", "log_alpha_m", "log_alpha_v")}
    snaps = {k: [] for k in NETS}
    moms = {"%s_%s" % (nm, w): [] for nm in NETS[:3] for w in ("m", "v")}
    opt = {"actor": tr.actor_optimizer, "critic_1": tr.critic_1_optimizer, "critic_2": tr.critic_2_optimizer}
    try:
        for step in range(K):
            s, a, r, s2, d = synth(rng)
            with torch.no_grad():
                rec["probs"].append(tr.actor(torch.tensor(s)).numpy().astype(np.float32))
            for k, v in zip(("s", "a", "r", "s2", "d"), (s, a, r, s2, d)):
                rec[k].append(v)
            mse_seen.clear()
            td = {"states": s.tolist(), "actions": a.tolist(), "next_states": s2.tolist(), "rewards": r.tolist(), "dones": d.tolist()}
            res = tr.update(td)
            assert len(mse_seen) == 2, mse_seen
            rec["actor_loss"].append(float(res["loss"]))
            rec["critic_1_loss"].append(mse_seen[0]); rec["critic_2_loss"].append(mse_seen[1])
            st = tr.log_alpha_optimizer.state[tr.log_alpha]
            rec["log_alpha"].append(tr.log_alpha.item())
            rec["log_alpha_m"].append(float(st["exp_avg"])); rec["log_alpha_v"].append(float(st["exp_avg_sq"]))
            for nm in NETS:
                snaps[nm].append(flat(getattr(tr, nm).state_dict().values())[idx])
            for nm, o in opt.items():
                ps = list(getattr(tr, nm).parameters())
                moms[nm + "_m"].append(flat([o.state[p]["exp_avg"] for p in ps])[idx])
                moms[nm + "_v"].append(flat([o.state[p]["exp_avg_sq"] for p in ps])[idx])
    finally:
        F.mse_loss = orig_mse
    for k, v in rec.items():
        out["sacd_" + k] = np.asarray(v, np.int32 if k == "a" else np.float32)
    for k, v in list(snaps.items()) + list(moms.items()):
        out["sacd_" + k] = np.stack(v)
    np.savez_compressed(os.path.join(HERE, "sac_discrete_golden.npz"), **out)
    print("sac discrete: P", out["sacd_actor0"].size, "sampled", idx.size, "actor losses", rec["actor_loss"], "critic losses",
          rec["critic_1_loss"], rec["critic_2_loss"], "log_alpha", rec["log_alpha"])


if __name__ == "__main__":
    main()
