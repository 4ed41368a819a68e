"""Grouped SAC learners (uavrl_sac_create_trainers): G independent SAC trainers in one handle, and the reference's actor
aggregation Federated_Learning_AC across them (uavrl_sac_federate_actors).  The defining property is checked bit for bit:
trainer g computes exactly what a stand-alone SacLearner with its parameters and alpha, seed + g, replay_capacity / G and
lockstep_envs / G computes -- act passes, explicit updates, ring-sampled updates and the whole lockstep loop."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fl_restatement import federate_actors
from gpu_util import (DEV, CountTransfers, assert_sac_trainers_equal, assert_same, city_and_params, dev, distinct_alphas, env_dict,
                      env_plugin, make_env, sac, sac_standalone_like)
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

G = 4
OBS, A = 100, 2
SAC_XML = ("Trainer_SAC_B200.xml", "UAV_continuous_B200.xml")     # the plug-in tests' trainer and agent: continuous step


def states(rng, n):
    return rng.uniform(-1, 1, (n, OBS)).astype(np.float32)


def batch(rng, n):
    return (states(rng, n), rng.uniform(-0.99, 0.99, (n, A)).astype(np.float32), rng.normal(0, 1, n).astype(np.float32),
            states(rng, n), (rng.random(n) < 0.1).astype(np.float32))


# ------------------------------------------------------------------ act
def test_act_blocks_equal_standalone():
    Ng = 1000                                             # ragged last tile
    rng = np.random.default_rng(1)
    S = sac(G)
    S.init_params(3)
    assert S.get_params(0).shape == (G, S.P[0]) and S.trainer_count() == G
    solo = [sac_standalone_like(S, g) for g in range(G)]
    obs = dev(states(rng, G * Ng))
    eps = dev(rng.normal(size=(G * Ng, A)).astype(np.float32))
    a_inj = S.act(obs, eps).cpu().numpy()                  # call 0 of every learner
    a_phi = S.act(obs).cpu().numpy()                       # call 1, Philox: keyed by seed + g and the trainer-local row
    for g, X in enumerate(solo):
        blk = slice(g * Ng, (g + 1) * Ng)
        assert_same(a_inj[blk], X.act(obs[blk].contiguous(), eps[blk].contiguous()).cpu().numpy(), "actions (eps), trainer %d" % g)
        assert_same(a_phi[blk], X.act(obs[blk].contiguous()).cpu().numpy(), "actions (Philox), trainer %d" % g)
    S.set_params(0, np.tile(S.get_params(0)[:1], (G, 1)))  # one actor everywhere: the blocks still draw different noise
    a_same = S.act(dev(np.tile(states(rng, Ng), (G, 1)))).cpu().numpy()
    assert not np.array_equal(a_same[:Ng], a_same[Ng:2 * Ng])


# ------------------------------------------------------------------ explicit updates
@pytest.mark.parametrize("B,ctas", [(64, 0), (200, 0), (200, 3)], ids=["B64", "B200", "B200-3ctas"])
def test_explicit_update_equals_standalone(B, ctas, monkeypatch):
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))    # the accumulating multi-tile path, per trainer
    rng = np.random.default_rng(B + ctas)
    S = sac(G)
    S.init_params(5)
    distinct_alphas(S, rng)
    solo = [sac_standalone_like(S, g) for g in range(G)]
    for step in range(4):
        s, a, r, s2, d = (dev(x) for x in batch(rng, G * B))
        injected = step % 2 == 1                              # Philox noise on steps 0 and 2, injected noise on 1 and 3
        e1 = dev(rng.normal(size=(G * B, A)).astype(np.float32)) if injected else None
        e2 = dev(rng.normal(size=(G * B, A)).astype(np.float32)) if injected else None
        losses = torch.zeros(4 * G, device=DEV)
        S.update_batch(s, a, r, s2, d, e1, e2, losses)
        solo_losses = []
        for g, X in enumerate(solo):
            blk = slice(g * B, (g + 1) * B)
            part = lambda t: None if t is None else t[blk].contiguous()  # noqa: E731
            l1 = torch.zeros(4, device=DEV)
            X.update_batch(part(s), part(a), part(r), part(s2), part(d), part(e1), part(e2), l1)
            solo_losses.append(l1.cpu().numpy())
        assert_sac_trainers_equal(S, solo, losses.cpu().numpy(), solo_losses)
    assert S.scalars()["epoch"] == 4 and S.scalars()["adam_step"] == 4


# ------------------------------------------------------------------ the lockstep ring
def grouped_and_pairs(env_golden, env27_golden, Ng, cap_g, seed, pool_seed):
    """A grouped learner on N = G Ng envs and, for every trainer, a stand-alone learner (seed + g, cap_g, Ng envs) on an env
    that starts from the same scenarios as the trainer's block."""
    N = G * Ng
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=pool_seed)
    env = make_env(env_golden, env27_golden, N, pool)
    env.reset(0)
    S = sac(G, seed=seed, replay_capacity=G * cap_g, lockstep_envs=N)
    S.init_params(1)
    distinct_alphas(S, np.random.default_rng(seed))
    pairs = []
    for g in range(G):
        e1 = make_env(env_golden, env27_golden, Ng, pool)
        e1.reset(g * Ng)
        pairs.append((e1, sac_standalone_like(S, g, seed=seed, replay_capacity=cap_g, lockstep_envs=Ng)))
    return env, S, pairs


def test_ring_sampled_updates_equal_standalone(env_golden, env27_golden):
    Ng, B, iters = 64, 64, 10
    env, S, pairs = grouped_and_pairs(env_golden, env27_golden, Ng, Ng * 16, 13, 3)
    engine.sac_train_run(env, S, iters, do_update=False)
    for e1, X in pairs:
        engine.sac_train_run(e1, X, iters, do_update=False)
    n_g = S.replay_size() // G
    assert n_g == iters * Ng and all(X.replay_size() == n_g for _, X in pairs)
    rng = np.random.default_rng(0)
    tape = np.stack([rng.choice(n_g, B, replace=False) for _ in range(G)]).astype(np.int32)
    for mode in ("tape", "philox"):
        losses = torch.zeros(4 * G, device=DEV)
        S.update_replay(dev(tape) if mode == "tape" else None, losses=losses)
        solo_losses = []
        for g, (_, X) in enumerate(pairs):
            l1 = torch.zeros(4, device=DEV)
            X.update_replay(dev(tape[g]) if mode == "tape" else None, losses=l1)
            solo_losses.append(l1.cpu().numpy())
        assert_sac_trainers_equal(S, [X for _, X in pairs], losses.cpu().numpy(), solo_losses)
    # the tape rows are the trainer's transitions: whole-ring index (k / Ng) N + g Ng + k % Ng
    k = tape[1].astype(np.int64)
    for x, y in zip(S.gather((k // Ng) * G * Ng + Ng + k % Ng), pairs[1][1].gather(k)):
        assert_same(x, y, "tape rows of trainer 1")


def test_lockstep_loop_equals_standalone_pairs(env_golden, env27_golden):
    Ng, iters = 384, 100
    cap_g = Ng * 40                                        # the ring wraps within the 100 iterations
    env, S, pairs = grouped_and_pairs(env_golden, env27_golden, Ng, cap_g, 11, 5)
    st = engine.sac_train_run(env, S, iters)
    assert st.env_steps == iters * G * Ng and st.updates > 0
    losses = []
    for e1, X in pairs:
        s1 = engine.sac_train_run(e1, X, iters)
        assert s1.updates == st.updates
        losses.append(np.float32(s1.last_loss))
    assert_sac_trainers_equal(S, [X for _, X in pairs])
    assert np.float32(st.last_loss) == np.float32(sum(float(x) for x in losses) / G)
    sg = env.get_state()
    n_g = S.replay_size() // G
    assert n_g == 40 * Ng                                  # full: the ring wrapped
    for g, (e1, X) in enumerate(pairs):
        s1 = e1.get_state()
        for k in sg:
            assert_same(sg[k][g * Ng:(g + 1) * Ng], s1[k], "env state %s, block %d" % (k, g))
        assert X.replay_size() == n_g
        k = np.arange(n_g, dtype=np.int64)
        ring_g = S.gather((k // Ng) * G * Ng + g * Ng + k % Ng)
        for x, y, what in zip(ring_g, X.gather(k), ("s", "a", "r", "s2", "d")):
            assert_same(x, y, "ring %s, trainer %d" % (what, g))
    # one more ring-sampled update: every trainer's own loss slots against its pair's losses
    out = torch.zeros(4 * G, device=DEV)
    S.update_replay(losses=out)
    solo_losses = []
    for _, X in pairs:
        l1 = torch.zeros(4, device=DEV)
        X.update_replay(losses=l1)
        solo_losses.append(l1.cpu().numpy())
    assert_sac_trainers_equal(S, [X for _, X in pairs], out.cpu().numpy(), solo_losses)


# ------------------------------------------------------------------ entry points, refusals, round trips
def test_refusals_round_trips_and_one_trainer():
    for bad in (0, 65536):                                 # one grid row per trainer: gridDim.y <= 65535
        with pytest.raises(engine.UavrlError, match="n_trainers must be in"):
            sac(bad)
    with pytest.raises(engine.UavrlError, match="multiple of n_trainers"):
        sac(3, lockstep_envs=64)
    with pytest.raises(engine.UavrlError, match="replay_capacity / n_trainers"):
        sac(8, replay_capacity=7, lockstep_envs=64)
    S = sac(G, lockstep_envs=64)
    assert S.trainer_count() == G
    x = torch.zeros((6, OBS), device=DEV)
    one = torch.zeros(6, device=DEV)
    with pytest.raises(engine.UavrlError, match="multiple of the trainer count"):
        S.act(x)
    with pytest.raises(engine.UavrlError, match="multiple of the trainer count"):
        S.update_batch(x, torch.zeros((6, A), device=DEV), one, x, one)
    x4, a4, o4 = x[:4], torch.zeros((4, A), device=DEV), one[:4]
    with pytest.raises(ValueError, match="4 trainers writes 16 losses"):
        S.update_batch(x4, a4, o4, x4, o4, losses=torch.zeros(4, device=DEV))
    with pytest.raises(ValueError, match="4 trainers writes 16 losses"):
        S.update_replay(losses=torch.zeros(15, device=DEV))
    rng = np.random.default_rng(0)
    for role in range(11):                                 # [G][P] round trip of every writable role
        p = rng.normal(0, 1, (G, S.P[role] if role < 5 else S.P[(role - 5) % 3])).astype(np.float32)
        S.set_params(role, p)
        assert_same(S.get_params(role), p, "round trip %d" % role)
    al = rng.normal(0, 1, (G, 3)).astype(np.float32)
    S.set_alpha(al)
    assert_same(S.alpha(), al, "alpha round trip")
    sc = S.scalars()                                       # trainer 0's triple
    assert (sc["log_alpha"], sc["la_m"], sc["la_v"]) == tuple(float(v) for v in al[0])
    S.set_scalars(-1.5, 0.25, 0.125, 9, 4)                 # one triple for every trainer
    assert_same(S.alpha(), np.tile(np.float32([-1.5, 0.25, 0.125]), (G, 1)), "set_scalars")
    assert (S.scalars()["epoch"], S.scalars()["adam_step"]) == (9, 4)
    with pytest.raises(ValueError, match="alpha triples"):
        S.set_alpha(np.zeros(3, np.float32))
    # G = 1 from the new entry point is the learner uavrl_sac_create makes
    L1 = sac(1)
    L0 = sac(1)
    _lib.lib().uavrl_sac_destroy(L0.h)
    L0.h = _lib.VP()
    engine.check(_lib.lib().uavrl_sac_create(_lib.C.byref(L0.cfg), _lib.C.byref(L0.h)))
    assert L1.get_params(0).shape == (L1.P[0],) and L1.alpha().shape == (1, 3)
    L1.init_params(4)
    for role in range(5):
        L0.set_params(role, L1.get_params(role))
    s, a, r, s2, d = (dev(v) for v in batch(rng, 256))
    for L in (L0, L1):
        L.update_batch(s, a, r, s2, d)
    assert_sac_trainers_equal(L1, [L0])
    assert_same(L0.act(s).cpu().numpy(), L1.act(s).cpu().numpy(), "actions")


# ------------------------------------------------------------------ Federated_Learning_AC
def test_federate_matches_reference_golden():
    g = np.load(os.path.join(GOLDEN, "fl_ac_golden.npz"))
    n = int(g["G"])
    S = sac(n)
    assert S.P[0] == g["actor0"].shape[1]
    S.set_params(0, g["actor0"])
    S.federate_actors()
    assert_same(S.get_params(0), g["actor1"], "actors after Federated_Learning_AC")


def test_federate_sums_actors_only_and_refreshes_images():
    rng = np.random.default_rng(4)
    S = sac(G)
    before = {}
    for role in range(11):                                 # full float32 mantissas: the summation order shows
        before[role] = (rng.normal(0, 0.1, (G, S.P[role] if role < 5 else S.P[(role - 5) % 3]))).astype(np.float32)
        if role >= 8:
            before[role] = np.abs(before[role])
        S.set_params(role, before[role])
    al = distinct_alphas(S, rng)
    S.set_scalars(*al[0], 5, 3)
    S.set_alpha(al)
    grads = [S.get_params(11 + r) for r in range(3)]
    S.federate_actors()
    torch.cuda.synchronize()
    want = federate_actors(before[0])
    assert_same(S.get_params(0), want, "every actor is the left-to-right sum")
    for role in range(1, 11):
        assert_same(S.get_params(role), before[role], "role %d untouched" % role)
    for r in range(3):
        assert_same(S.get_params(11 + r), grads[r], "gradient %d untouched" % r)
    assert_same(S.alpha(), al, "alpha untouched")
    assert (S.scalars()["epoch"], S.scalars()["adam_step"]) == (5, 3)
    # the actor images were refreshed: an act pass now equals stand-alone learners loaded with the summed actor
    Ng = 96
    obs = dev(states(rng, G * Ng))
    acts = S.act(obs).cpu().numpy()
    for g in range(G):
        X = sac(1, 7 + g)
        X.set_params(0, want[g])
        assert_same(acts[g * Ng:(g + 1) * Ng], X.act(obs[g * Ng:(g + 1) * Ng].contiguous()).cpu().numpy(), "act after federate, %d" % g)


def test_federate_one_trainer_keeps_actor():
    S = sac(1)
    S.init_params(2)
    p = S.get_params(0)
    obs = dev(states(np.random.default_rng(5), 64))
    e = dev(np.zeros((64, A), np.float32))
    a0 = S.act(obs, e).cpu().numpy()
    S.federate_actors()
    assert_same(S.get_params(0), p, "G = 1 actor")
    assert_same(S.act(obs, e).cpu().numpy(), a0, "G = 1 actions")


# ------------------------------------------------------------------ plug-ins
def test_env_plugin_one_sac_trainer_per_uav(tmp_path):
    """num_UAV = num_trainers = 8 with the shipped SAC trainer and the continuous step: run_eposide runs, save() writes the
    reference's three files per UAV, Load_Mod in a fresh env restores every trainer bit for bit, each moving every role's
    vector between host and device once whatever G is; Is_FL = Is_AC = FL_Loop = 1 leaves every actor equal to the sum."""
    with env_plugin(tmp_path) as mod:
        env = mod.PathPlan_City_B200(env_dict(*SAC_XML))
        tr = env.Trainer
        assert tr._learner.trainer_count() == 8 and tr.names == ["UAV_%d" % i for i in range(8)]
        with pytest.raises(ValueError, match="batch"):
            tr.get_action(np.zeros(100, np.float32))
        assert tr.get_action(np.zeros((8, 100), np.float32)).shape == (8, 2)
        info = env.run_eposide(0.3)
        assert info["updates"] > 0 and np.isfinite(info["loss"])
        n = CountTransfers(tr._learner)
        tr.save()
        assert (n.get, n.set) == (9, 0)
        env2 = mod.PathPlan_City_B200(env_dict(*SAC_XML))                     # Load_Mod in the constructor
        n = CountTransfers(env2.Trainer._learner)
        env2.Trainer.Load_Mod()
        assert (n.get, n.set) == (9, 11)
        # federated aggregation of the actors after every episode
        env3 = mod.PathPlan_City_B200(env_dict(*SAC_XML, Is_FL="1", Is_AC="1", FL_Loop="1"))
        L3 = env3.Trainer._learner
        seen = []
        fed = L3.federate_actors

        def spy():
            seen.append(L3.get_params(0))
            fed()
        L3.federate_actors = spy
        env3.run_eposide(0.3)
        assert len(seen) == 1
        assert_same(L3.get_params(0), federate_actors(seen[0]), "actors after the episode")
    files = sorted(os.listdir(tmp_path))
    assert files == sorted(["%s_SAC_UAV_%d.pth" % (k, i) for k in ("actor", "critic_1", "critic_2") for i in range(8)]), files
    ck = torch.load(os.path.join(tmp_path, "critic_2_SAC_UAV_5.pth"), weights_only=False)
    assert set(ck) == {"model", "optimizer", "epoch"}
    assert_same(ck["model"]["fc1.weight"].numpy().ravel(), tr._learner.get_params(2)[5][:64 * 102], "trainer 5 critic_2 fc1.weight")
    L, L2 = tr._learner, env2.Trainer._learner
    for role in (0, 1, 2, 5, 6, 7, 8, 9, 10):
        assert_same(L2.get_params(role), L.get_params(role), "restored role %d" % role)
    for role in (1, 2):
        assert_same(L2.get_params(role + 2), L.get_params(role), "target %d copies the critic" % role)
    assert (L2.scalars()["epoch"], L2.scalars()["adam_step"]) == (L.scalars()["epoch"], L.scalars()["adam_step"])


def test_env_plugin_skips_malformed_checkpoint(tmp_path, capsys):
    """Trainer 3's critic_1 file holds a renamed key.  As in the reference (SAC_Trainer.py:105-106), the constructor prints
    the error and carries on: trainer 3 keeps its fresh networks, targets and moments, every other trainer is restored bit
    for bit with its targets copying its critics."""
    with env_plugin(tmp_path) as mod:
        tr = mod.PathPlan_City_B200(env_dict(*SAC_XML)).Trainer                  # no files yet: fresh parameters
        L = tr._learner
        fresh = {r: L.get_params(r) for r in range(11)}
        rng = np.random.default_rng(5)
        saved = {r: rng.normal(0, 1, fresh[r].shape).astype(np.float32) for r in (0, 1, 2, 5, 6, 7, 8, 9, 10)}
        for r, x in saved.items():
            L.set_params(r, x)
        tr._set_counters(123, 45)
        tr.save()
        p = os.path.join(tmp_path, "critic_1_SAC_UAV_3.pth")
        ck = torch.load(p, weights_only=False)
        ck["model"] = {("fc3.weight" if k == "fc_out.weight" else k): t for k, t in ck["model"].items()}
        torch.save(ck, p)
        capsys.readouterr()
        L2 = mod.PathPlan_City_B200(env_dict(*SAC_XML)).Trainer._learner         # Load_Mod in the constructor
        out = capsys.readouterr().out
    assert "critic_1_SAC_UAV_3.pth holds" in out and "fc3.weight" in out, out
    for r in range(11):
        want = saved.get(r, saved.get(r - 2))                            # targets 3, 4 copy critics 1, 2
        for g in range(8):
            assert_same(L2.get_params(r)[g], fresh[r][g] if g == 3 else want[g], "role %d of trainer %d" % (r, g))
    assert (L2.scalars()["epoch"], L2.scalars()["adam_step"]) == (123, 45)
