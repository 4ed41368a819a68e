"""Prioritised replay on grouped learners (uavrl_per_enable_trainers): one SumTree per trainer.  The defining property is
checked bit for bit: trainer g with prioritised replay computes exactly what a stand-alone learner with prioritised replay, its
parameters, seed + g, replay_capacity / G and lockstep_envs / G computes -- sampled slots and weights, each tree's leaves,
total and beta, parameters, Adam moments, gradient and loss.  The sampler is also checked per trainer against the CPU oracle
of the reference's SumTree, and the trees against each other (a write to one trainer leaves the others untouched)."""
import os

import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import (DEV, PER_MAX, ROOT, assert_same, assert_trainers_equal, assert_trees_equal, city_and_params, env_dict,
                      learner, make_env, n_sm)  # noqa: F401  (module fixture)
from shapes import SHIPPED
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu
P0 = float(np.float32(0.01) ** np.float32(0.6))        # priority of a transition stored without an error


def generated_env(env_golden, env27_golden, n, pool=256):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=True)
    env.generate_pool(pool, seed=2)
    env.reset(0)
    return env


CASES = [  # algo, shape, tensor cores, per-trainer batch, loss
    ("dqn", engine.ALGO_DQN, SHIPPED[0], True, 64, "mse"),
    ("ddqn", engine.ALGO_DDQN, SHIPPED[0], True, 64, "mse"),
    ("dueling", engine.ALGO_DUELING, SHIPPED[2], True, 64, "mse"),
    ("dqn-fp32", engine.ALGO_DQN, SHIPPED[0], False, 64, "mse"),
    ("ddqn-fp32", engine.ALGO_DDQN, SHIPPED[0], False, 64, "mse"),
    ("dueling-fp32", engine.ALGO_DUELING, SHIPPED[2], False, 64, "mse"),
    ("ddqn-huber", engine.ALGO_DDQN, SHIPPED[0], True, 64, "huber"),
    ("ddqn-B9000", engine.ALGO_DDQN, SHIPPED[0], True, 9000, "mse"),          # 64-row tiles, TD targets in separate passes
    ("dqn-fp32-B9000", engine.ALGO_DQN, SHIPPED[0], False, 9000, "mse"),
]


@pytest.mark.parametrize("algo,shape,tc,B,loss", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_lockstep_loop_with_per_equals_standalone_pairs(env_golden, env27_golden, algo, shape, tc, B, loss):
    G, Ng, iters = 4, 384, 100
    N, cap_g = G * Ng, Ng * 40                          # the ring wraps within the 100 iterations
    n_slots = (cap_g // Ng + 1) * Ng                    # trainer-local slots: ring frames x Ng
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=5)
    env = make_env(env_golden, env27_golden, N, pool)
    env.reset(0)
    kw = dict(algo=algo, update_loop=3, batch_size=B, loss=loss)
    Lg = learner(shape, G, seed=11, replay_capacity=G * cap_g, lockstep_envs=N, **kw)
    Lg.init_params(1)
    Lg.per_enable_trainers()
    Lg.set_tensor_cores(tc)
    if tc:                                               # both places trainer_src hands out the weight / |Q - y| rows
        r = Lg.route(B)
        assert r["train_rows"] == (32 if B == 64 else 64)
        assert r["td_fused"] if (B == 64 and algo == engine.ALGO_DDQN) else (B == 64 or not r["td_fused"])
    st = engine.train_run(env, Lg, iters, eps=0.2)
    assert st.episodes_ended == 0 and st.updates > 0
    pairs, losses = [], []
    for g in range(G):
        e1 = make_env(env_golden, env27_golden, Ng, pool)
        e1.reset(g * Ng)
        L1 = learner(shape, 1, seed=11 + g, replay_capacity=cap_g, lockstep_envs=Ng, **kw)
        L1.init_params(1 + g)
        L1.per_enable()
        L1.set_tensor_cores(tc)
        s1 = engine.train_run(e1, L1, iters, eps=0.2)
        assert s1.updates == st.updates
        pairs.append((e1, L1)); losses.append(np.float32(s1.last_loss))
    solo = [L1 for _, L1 in pairs]
    assert_trainers_equal(Lg, solo)
    assert_trees_equal(Lg, solo, n_slots)
    assert np.float32(st.last_loss) == np.float32(sum(float(x) for x in losses) / G)
    # one more ring-sampled update: every trainer's own loss slot, tree and parameters against its pair's
    loss_g = torch.zeros(G, device=DEV)
    Lg.update(loss=loss_g)
    solo_loss = []
    for L1 in solo:
        l1 = torch.zeros(1, device=DEV)
        L1.update(loss=l1)
        solo_loss.append(l1.cpu().numpy())
    assert_trainers_equal(Lg, solo, loss_g.cpu().numpy(), solo_loss)
    assert_trees_equal(Lg, solo, n_slots)
    # the sampler on its own: slots and weights of every trainer
    sg, wg = Lg.per_sample(B)
    for g, L1 in enumerate(solo):
        s1, w1 = L1.per_sample(B)
        assert_same(sg[g].cpu().numpy(), s1.cpu().numpy(), "sampled slots of trainer %d" % g)
        assert_same(wg[g].cpu().numpy(), w1.cpu().numpy(), "weights of trainer %d" % g)
    for e1, L1 in pairs:
        e1.close(); L1.close()
    env.close(); Lg.close()


def filled_learner(env_golden, env27_golden, G, Ng, frames, iters, **kw):
    """A grouped learner with prioritised replay whose ring holds `iters` transition groups (no updates)."""
    env = generated_env(env_golden, env27_golden, G * Ng)
    L = learner(SHIPPED[0], G, replay_capacity=G * Ng * frames, lockstep_envs=G * Ng, **kw)
    L.init_params(0)
    L.per_enable_trainers()
    engine.train_run(env, L, iters, eps=0.5, do_update=False)
    assert L.replay_size() == iters * G * Ng
    return env, L, (frames + 1) * Ng


def test_sampler_per_trainer_vs_oracle(env_golden, env27_golden, n_sm):
    """300 trainers (grid y = 300), B = 5000 draws each -- more than one trainer's grid-stride width of 8 x (4 x SMs) warps.
    Dyadic priorities (every partial sum exact) whose totals differ by up to 2^11 between trainers, one trainer with a single
    non-zero leaf: every trainer's slots are the oracle's on that trainer's priorities, its weights are normalised by its
    own maximum, and beta follows the shared schedule.  A shared total, a shared maximum or a wrong tree offset fails."""
    G, Ng, B = 300, 4, 5000
    assert B > 8 * 4 * n_sm
    env, L, cap = filled_learner(env_golden, env27_golden, G, Ng, 600, 10)
    rng = np.random.default_rng(9)
    prio = np.ldexp(rng.integers(1, 4096, (G, cap)).astype(np.float64), -10)
    prio *= np.ldexp(1.0, rng.integers(-1, 11, G))[:, None]
    prio[rng.random((G, cap)) < 0.05] = 0.0
    lone = 123
    prio[lone] = 0.0
    prio[lone, 777] = 37.0
    slots = torch.arange(cap, dtype=torch.int32, device=DEV).repeat(G, 1)
    L.per_set_priorities(slots, torch.tensor(prio, device=DEV))
    leaves, totals, beta0 = L.per_state(cap)
    assert np.array_equal(leaves, prio) and np.array_equal(totals, prio.sum(1))
    u = rng.random((G, B))
    s, w = L.per_sample(B, torch.tensor(u, device=DEV))
    s, w = s.cpu().numpy().astype(np.int64), w.cpu().numpy()
    assert s.shape == w.shape == (G, B)
    for g in range(G):
        per = O.OraclePer(cap)
        per.add(prio[g])
        idx_o, w_o, beta_o = per.sample(u[g])
        assert np.array_equal(s[g] + cap - 1, idx_o), g
        np.testing.assert_allclose(w[g], w_o, rtol=2e-6, err_msg="trainer %d" % g)
    assert (s[lone] == 777).all() and (w[lone] == 1.0).all()
    assert L.per_state(cap)[2] == beta_o
    env.close(); L.close()


@pytest.mark.parametrize("clip", [True, False], ids=["batch_update", "push"])
def test_set_errors_touches_one_tree(env_golden, env27_golden, clip):
    """per_set_errors that changes only trainer 2's errors (the other rows rewrite the errors they already hold) leaves every
    other trainer's leaves and total bitwise unchanged, and trainer 2's leaves follow the rule."""
    G, Ng, g = 6, 4, 2
    env, L, cap = filled_learner(env_golden, env27_golden, G, Ng, 300, 5)
    rng = np.random.default_rng(4)
    e0 = rng.uniform(0, 2, (G, cap)).astype(np.float32)
    L.per_set_errors(torch.arange(cap, dtype=torch.int32, device=DEV).repeat(G, 1), torch.tensor(e0, device=DEV), clip=clip)
    leaves0, totals0, _ = L.per_state(cap)
    pick = np.sort(rng.choice(cap, 100, replace=False))
    e1 = e0[:, pick].copy()
    e1[g] = rng.uniform(0, 2, 100).astype(np.float32)
    L.per_set_errors(torch.tensor(np.tile(pick, (G, 1)).astype(np.int32), device=DEV), torch.tensor(e1, device=DEV), clip=clip)
    leaves1, totals1, _ = L.per_state(cap)
    for h in range(G):
        if h != g:
            assert_same(leaves1[h], leaves0[h], "leaves of trainer %d" % h)
            assert_same(totals1[h:h + 1], totals0[h:h + 1], "total of trainer %d" % h)
    e = np.abs(e1[g]) + np.float32(0.01)
    if clip:
        e = np.minimum(e, np.float32(1.0))
    np.testing.assert_allclose(leaves1[g, pick], np.power(e, np.float32(0.6)).astype(np.float64), rtol=3e-7, atol=0)
    rest = np.setdiff1d(np.arange(cap), pick)
    assert_same(leaves1[g, rest], leaves0[g, rest], "untouched leaves of trainer %d" % g)
    assert not np.array_equal(leaves1[g], leaves0[g])
    assert abs(totals1[g] - leaves1[g].sum()) <= 1e-12 * totals1[g]
    env.close(); L.close()


def test_lockstep_commit_layout(env_golden, env27_golden):
    """16 trainers after a lockstep loop: in every trainer's tree exactly one frame is empty (the head, the same frame for
    every trainer), stored transitions carry priorities in [eps^alpha, 1], sampled ones were re-prioritised, and each total is
    the sum of that trainer's leaves."""
    G, Ng, F = 16, 64, 12
    env = generated_env(env_golden, env27_golden, G * Ng, pool=512)
    L = learner(SHIPPED[0], G, seed=1, algo=engine.ALGO_DDQN, batch_size=Ng, replay_capacity=G * Ng * F, lockstep_envs=G * Ng,
                update_loop=3)
    L.init_params(0)
    L.per_enable_trainers()
    st = engine.train_run(env, L, 40, eps=0.3)
    assert st.updates == 39 and np.isfinite(st.last_loss)
    leaves, totals, beta = L.per_state((F + 1) * Ng)
    assert abs(beta - min(1.0, 0.4 + 0.001 * st.updates)) < 1e-12
    heads = set()
    for g in range(G):
        lv = leaves[g].reshape(F + 1, Ng)
        empty = np.where((lv == 0).all(1))[0]
        assert len(empty) == 1, g
        heads.add(int(empty[0]))
        filled = np.delete(lv, empty[0], axis=0)
        assert filled.min() >= P0 * (1 - 1e-6) and filled.max() <= 1.0 + 1e-6
        assert (np.abs(filled - P0) > 1e-9).sum() > Ng              # sampled transitions were re-prioritised
        assert abs(totals[g] - leaves[g].sum()) <= 1e-9 * totals[g]
    assert len(heads) == 1
    env.close(); L.close()


@pytest.mark.parametrize("G", [1, 4])
def test_lockstep_restart_clears_trees(env_golden, env27_golden, G):
    """lockstep_restart after updates have re-prioritised leaves empties the ring and every tree (leaves and totals 0, beta
    kept); the first iteration after it gives exactly one frame of Ng slots per tree the push priority eps^alpha."""
    Ng, F = 64, 12
    cap = (F + 1) * Ng
    env = generated_env(env_golden, env27_golden, G * Ng, pool=512)
    L = learner(SHIPPED[0], G, seed=1, algo=engine.ALGO_DDQN, batch_size=Ng, replay_capacity=G * Ng * F, lockstep_envs=G * Ng,
                update_loop=3)
    L.init_params(0)
    L.per_enable_trainers()
    st = engine.train_run(env, L, 20, eps=0.3)
    assert st.updates == 19
    leaves, _, beta = L.per_state(cap)
    leaves = leaves.reshape(G, cap)
    for g in range(G):
        assert (np.abs(leaves[g][leaves[g] != 0] - P0) > 1e-9).sum() > Ng, g     # sampled transitions were re-prioritised
    L.lockstep_restart()
    env.reset(0)
    assert L.replay_size() == 0
    leaves, totals, beta1 = L.per_state(cap)
    assert not leaves.any() and not np.any(totals)
    assert beta1 == beta
    st = engine.train_run(env, L, 1, eps=0.3)
    assert st.updates == 0 and L.replay_size() == G * Ng
    leaves = L.per_state(cap)[0].reshape(G, F + 1, Ng)
    for g in range(G):
        full = np.where(leaves[g].any(1))[0]
        assert len(full) == 1, g
        assert (leaves[g, full[0]] != 0).all()
        np.testing.assert_allclose(leaves[g, full[0]], P0, rtol=1e-6, atol=0)
    env.close(); L.close()


def test_one_trainer_and_refusals(env_golden, env27_golden):
    # G = 1: per_enable_trainers is per_enable
    runs = []
    for enable in ("per_enable", "per_enable_trainers"):
        env = generated_env(env_golden, env27_golden, 256)
        L = learner(SHIPPED[0], 1, seed=3, algo=engine.ALGO_DDQN, batch_size=64, replay_capacity=256 * 12, lockstep_envs=256)
        L.init_params(0)
        getattr(L, enable)()
        engine.train_run(env, L, 30, eps=0.3)
        runs.append((env, L))
    (e0, L0), (e1, L1) = runs
    assert_trainers_equal(L1, [L0])
    leaves1, total1, beta1 = L1.per_state(256 * 13)
    leaves0, total0, beta0 = L0.per_state(256 * 13)
    assert isinstance(total1, float) and leaves1.shape == (256 * 13,)
    assert_same(leaves1, leaves0, "leaves")
    assert total1 == total0 and beta1 == beta0
    for e, L in runs:
        e.close(); L.close()
    # refused once a transition is stored
    env = generated_env(env_golden, env27_golden, 64)
    Lg = learner(SHIPPED[0], 4, replay_capacity=64 * 8, lockstep_envs=64)
    engine.train_run(env, Lg, 1, eps=0.5, do_update=False)
    with pytest.raises(engine.UavrlError, match="before the first transition"):
        Lg.per_enable_trainers()
    # today's refusals on a grouped learner are unchanged
    with pytest.raises(engine.UavrlError, match="prioritised replay is not available on a learner with several trainers"):
        Lg.per_enable()
    x, one = torch.zeros((4, SHIPPED[0][0]), device=DEV), torch.zeros(4, device=DEV)
    with pytest.raises(engine.UavrlError, match="update_batch_per"):
        Lg.update_batch_per(x, one.int(), one, x, one)
    env.close(); Lg.close()
    # grouped prioritised replay samples the lockstep ring
    with pytest.raises(engine.UavrlError, match="lockstep ring"):
        learner(SHIPPED[0], 4).per_enable_trainers()
    # cap_g = ring_frames x Ng: the limit itself is accepted, one slot more is refused before anything is allocated
    small = [4, [32], 5, False]
    L = learner(small, 2, replay_capacity=2 * 4 * (PER_MAX // 4 - 1), lockstep_envs=8)
    L.per_enable_trainers()
    leaves, totals, _ = L.per_state(PER_MAX)
    assert leaves.shape == (2, PER_MAX) and not leaves.any() and not totals.any()
    L.close()
    L = learner(small, 2, replay_capacity=2 * 5 * ((PER_MAX + 1) // 5 - 1), lockstep_envs=10)
    with pytest.raises(engine.UavrlError, match="at most 4194304 slots"):
        L.per_enable_trainers()
    with pytest.raises(engine.UavrlError, match="not enabled"):
        L.per_state(1)
    L.close()


def test_env_plugin_prioritised_replay_per_trainer(tmp_path):
    """num_UAV = num_trainers = 8 with the DDQN Trainer XML and IsPriority_Replay = 1: every trainer gets its own tree,
    run_eposide trains, every tree holds re-prioritised leaves; with Is_FL = 1, FL_Loop = 1 the aggregation runs and leaves
    every tree as it was; save() / Load_Mod round-trip the trainers."""
    import importlib
    cwd = os.getcwd()
    os.chdir(ROOT)
    try:
        mod = importlib.import_module("uavrl_b200.plugins.PathPlan_City_B200")
        orig = mod.XML2Dict

        def patched(path):
            d = orig(path)
            if "Trainer" in d and isinstance(d["Trainer"], dict):
                d["Trainer"].update(Batch_Size="16", replay_size="512", save_loop="0", model_path=str(tmp_path),
                                    IsPriority_Replay="1")
            return d
        mod.XML2Dict = patched
        try:
            env = mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml", Is_FL="1", FL_Loop="1"))
            tr = env.Trainer
            assert tr._learner.trainer_count() == 8 and tr.IsPriority_Replay
            calls = []
            fl = env.Federated_Learning_choice

            def counted():
                leaves0, totals0, beta0 = tr._learner.per_state(n_slots)
                p0 = tr._learner.get_params(0)
                fl()
                leaves1, totals1, beta1 = tr._learner.per_state(n_slots)
                assert_same(leaves1, leaves0, "leaves across the aggregation")
                assert_same(totals1, totals0, "totals across the aggregation")
                assert beta1 == beta0
                calls.append(not np.array_equal(p0, tr._learner.get_params(0)))
            env.Federated_Learning_choice = counted
            L = tr._learner
            n_slots = (512 + 1) * 1             # trainer-local slots: (replay_size / Ng + 1) ring frames x Ng = 1 env per trainer
            info = env.run_eposide(0.3)
            assert info["updates"] > 0 and np.isfinite(info["loss"])
            assert calls == [True]                                          # aggregated once, q_local changed, trees kept
            leaves, totals, _ = L.per_state(n_slots)
            for g in range(8):
                stored = leaves[g][leaves[g] > 0]
                assert stored.size > 0 and (np.abs(stored - P0) > 1e-9).any(), g
                assert abs(totals[g] - leaves[g].sum()) <= 1e-9 * totals[g]
            tr.save()
            env2 = mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml"))                       # Load_Mod in the constructor
            assert env2.Trainer._learner.per_state(n_slots)[0].shape == (8, n_slots)
        finally:
            mod.XML2Dict = orig
    finally:
        os.chdir(cwd)
    for which in range(4):
        assert_same(env2.Trainer._learner.get_params(which), tr._learner.get_params(which), "restored vector %d" % which)
    assert env2.Trainer._learner.counters() == tr._learner.counters()
