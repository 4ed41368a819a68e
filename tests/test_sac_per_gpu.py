"""Prioritised replay for the SAC learner (include/uavrl.h, uavrl_sac_per_enable): the weighted critic kernel against the float64
restatement, the integrated ring update against its composition from the public calls, grouped trainers against stand-alone
twins (trees included), the data-parallel forms, the refusals, the launch counts and the plug-ins."""
import numpy as np
import pytest
import torch

from gpu_util import (DEV, assert_sac_trainers_equal, assert_same, city_and_params, dev, distinct_alphas, env_dict, env_plugin,
                      make_env, sac, sac_standalone_like)
from replay_restatement import Ring, per_uniforms
from sac_restatement import HP, check_step, draw_batch, init_state, near_decision, read_state
from sac_weighted_restatement import sac_update64_weighted
from shapes import SAC_SHAPES, sac_shape_id
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

OBS, A = 100, 2
SAC_XML = ("Trainer_SAC_B200.xml", "UAV_continuous_B200.xml")


def load_state(S, st):
    for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v")):
        S.set_params(role, st[k])
    S.set_scalars(st["log_alpha"], st["la_m"], st["la_v"], epoch=st["step"], adam_step=st["step"])


def weights(rng, B):
    w = rng.uniform(0, 1, B).astype(np.float32)
    w[:2], w[2:4] = 0.0, 1.0
    return w


def weighted_batch(rng, st, B, obs, hid, bound):
    """clean_batch for the weighted update (its critic step, and so the actor leg, depends on the weights): rows near a
    decision point of their own are drawn again whole, then rows near one in the actor leg get fresh eps_cur.  Returns the
    batch, its weights and the float64 step."""
    batch, w = list(draw_batch(rng, B, obs, bound)), weights(rng, B)
    for _ in range(40):
        new, out = sac_update64_weighted(st, *batch, obs, hid, bound, w)
        near, near_actor = near_decision(out)
        if near.any():
            for x, y in zip(batch, draw_batch(rng, int(near.sum()), obs, bound)):
                x[near] = y
        elif near_actor.any():
            batch[6][near_actor] = rng.normal(size=(int(near_actor.sum()), A))
        else:
            return batch, w, new, out
    raise AssertionError("could not draw a weighted batch clear of the decision points")


# ------------------------------------------------------------------ 1. the weighted kernel against float64
LEGS = {"B64": (64, 0), "B200": (200, 0), "B200-3ctas": (200, 3)}


@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
@pytest.mark.parametrize("leg", list(LEGS))
def test_weighted_update_vs_float64(shape, leg, monkeypatch):
    """update_batch_per, 3 chained updates: every state word, loss and gradient within check_step's bounds of
    sac_update64_weighted, and abs_err_out within 1e-5 of its terms' magnitude of the restated e_b.  A grouped learner (G = 4)
    on the same kind of batches equals four stand-alone learners bit for bit, e_b included."""
    obs, hid, bound, _ = shape
    B, ctas = LEGS[leg]
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))
    rng = np.random.default_rng(obs * 1000 + hid + B)
    st = init_state(rng, obs, hid)
    S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, **HP)
    load_state(S, st)
    losses = torch.zeros(4, device=DEV)
    for step in range(3):
        prev = read_state(S)
        batch, w, new, out = weighted_batch(rng, prev, B, obs, hid, bound)
        s, a, r, s2, d, e1, e2 = batch
        ae = torch.full((B,), -1.0, device=DEV)
        S.update_batch_per(dev(s), dev(a), dev(r), dev(s2), dev(d), dev(w), ae, dev(e1), dev(e2), losses)
        torch.cuda.synchronize()
        check_step(S, prev, new, out, losses.cpu().numpy().astype(np.float64), (leg, step))
        err = np.abs(ae.cpu().numpy() - out["abs_err"]) - (1e-5 * out["abs_err_scale"] + 1e-5 * out["abs_err"])
        assert (err <= 0).all(), (leg, step, "e_b", float(err.max()))
    S.close()
    # G = 4: trainer g is its stand-alone twin, its e_b block included
    G = 4
    Sg = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, trainers=G, seed=3, **HP)
    Sg.init_params(2)
    distinct_alphas(Sg, rng)
    solo = [sac_standalone_like(Sg, g, seed=3, obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B) for g in range(G)]
    for step in range(2):
        s, a, r, s2, d = (dev(rng.normal(0, 1, sh).astype(np.float32)) for sh in ((G * B, obs), (G * B, A), (G * B,), (G * B, obs), (G * B,)))
        d = (d > 1.0).float()
        w = dev(np.concatenate([weights(rng, B) for _ in range(G)]))
        ae, lg = torch.zeros(G * B, device=DEV), torch.zeros(4 * G, device=DEV)
        Sg.update_batch_per(s, a, r, s2, d, w, ae, None, None, lg)
        solo_losses = []
        for g, X in enumerate(solo):
            blk = slice(g * B, (g + 1) * B)
            a1, l1 = torch.zeros(B, device=DEV), torch.zeros(4, device=DEV)
            X.update_batch_per(*(t[blk].contiguous() for t in (s, a, r, s2, d, w)), a1, None, None, l1)
            solo_losses.append(l1.cpu().numpy())
            assert_same(ae[blk].cpu().numpy(), a1.cpu().numpy(), "e_b of trainer %d" % g)
        assert_sac_trainers_equal(Sg, solo, lg.cpu().numpy(), solo_losses)


# ------------------------------------------------------------------ helpers on the ring
def ring_learners(env_golden, env27_golden, n, cap, seed=7, twins=2, trainers=1, pool_seed=3):
    """`twins` learners with prioritised replay, identical parameters and alpha, each on its own env started from the same
    scenarios (so their rings and trees fill identically)."""
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, n, max_subgoals=64).make_scenarios(n, seed=pool_seed)
    out = []
    for _ in range(twins):
        env = make_env(env_golden, env27_golden, n, pool)
        env.reset(0)
        S = sac(trainers, seed=seed, replay_capacity=cap, lockstep_envs=n)
        S.init_params(1)
        distinct_alphas(S, np.random.default_rng(seed))
        S.per_enable()
        out.append((env, S))
    return out


def trees_equal(S, X, what):
    n = S.tree_slots()
    l0, t0, b0 = S.per_state(n)
    l1, t1, b1 = X.per_state(n)
    assert_same(l0, l1, what + ": leaves")
    assert_same(np.atleast_1d(t0), np.atleast_1d(t1), what + ": totals")
    assert b0 == b1, what + ": beta"


def learners_equal(S, X, what, l0=None, l1=None):
    for role in range(14):
        assert_same(S.get_params(role), X.get_params(role), "%s: role %d" % (what, role))
    assert_same(S.alpha(), X.alpha(), what + ": alpha")
    assert S.scalars()["epoch"] == X.scalars()["epoch"] and S.scalars()["adam_step"] == X.scalars()["adam_step"]
    if l0 is not None:
        assert_same(l0.cpu().numpy(), l1.cpu().numpy(), what + ": losses")
    trees_equal(S, X, what)


def composed_update(X, ring, calls, B, losses):
    """One prioritised ring update of X from its public parts: per_sample with the restated uniforms, the sampled rows
    gathered, update_batch_per with their weights at the same epoch, then per_set_errors(clip)."""
    u = per_uniforms(X.cfg.seed, calls, B)
    slots, w = X.per_sample(B, dev(u, torch.float64))
    sl = slots.cpu().numpy().astype(np.int64)
    Ng = ring.Ng
    J = ((sl // Ng - ring.oldest()) % ring.ring_frames) * ring.N + sl % Ng      # trainer-local slot -> logical index (G = 1)
    s, a, r, s2, d = X.gather(J)
    ae = torch.zeros(B, device=DEV)
    X.update_batch_per(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), w, ae, None, None, losses)
    X.per_set_errors(slots, ae, clip=True)
    return sl


# ------------------------------------------------------------------ 2. the integrated update is its composition
def test_update_replay_is_its_composition(env_golden, env27_golden):
    """update_replay with the trees on equals, bit for bit, per_sample (restated uniforms) -> gather -> update_batch_per ->
    per_set_errors on a twin: parameters, moments, alpha, losses, leaves, totals and beta, over 3 updates after a wrap."""
    N, B = 128, 64
    cap = N * 6
    (e0, S), (e1, X) = ring_learners(env_golden, env27_golden, N, cap)
    iters = 9                                                   # the ring (7 frames) wraps
    engine.sac_train_run(e0, S, iters, do_update=False)
    engine.sac_train_run(e1, X, iters, do_update=False)
    ring = Ring(cap, N)
    for _ in range(iters):
        ring.commit()
    trees_equal(S, X, "after the fill")
    leaves0, _, beta0 = S.per_state(S.tree_slots())
    for k in range(3):
        l0, l1 = torch.zeros(4, device=DEV), torch.zeros(4, device=DEV)
        S.update_replay(losses=l0)
        sl = composed_update(X, ring, k, B, l1)
        torch.cuda.synchronize()
        learners_equal(S, X, "update %d" % k, l0, l1)
    leaves, _, beta = S.per_state(S.tree_slots())
    assert beta > beta0 and (leaves[sl] != leaves0[sl]).any()


# ------------------------------------------------------------------ 3. the grouped lockstep loop
def test_grouped_loop_equals_standalone_trees(env_golden, env27_golden):
    """sac_train_run with G = 4 and prioritised replay over iterations that wrap the ring: every trainer equals its stand-alone
    twin (seed + g, capacity / G, envs / G, its own trees) bit for bit, tree and beta included; a commit gives the newest frame
    Ng leaves of the float32 eps^alpha and the frame the ring drops 0."""
    G, Ng = 4, 96
    cap_g = Ng * 8
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, G * Ng, max_subgoals=64).make_scenarios(G * Ng, seed=5)
    env = make_env(env_golden, env27_golden, G * Ng, pool)
    env.reset(0)
    S = sac(G, seed=11, replay_capacity=G * cap_g, lockstep_envs=G * Ng)
    S.init_params(1)
    distinct_alphas(S, np.random.default_rng(2))
    pairs = []
    for g in range(G):
        e1 = make_env(env_golden, env27_golden, Ng, pool)
        e1.reset(g * Ng)
        X = sac_standalone_like(S, g, seed=11, replay_capacity=cap_g, lockstep_envs=Ng)
        X.per_enable()
        pairs.append((e1, X))
    S.per_enable()
    n = S.tree_slots()
    assert n == pairs[0][1].tree_slots() == 9 * Ng
    ring = Ring(G * cap_g, G * Ng, G)
    p_new = None
    for it in range(14):                                        # updates start at iteration 2; the 9-frame ring wraps
        st = engine.sac_train_run(env, S, 1)
        for e1, X in pairs:
            engine.sac_train_run(e1, X, 1)
        f = ring.head
        ring.commit()
        leaves, _, _ = S.per_state(n)
        if st.updates == 0:                                     # the commit alone: frame f new, frame f + 1 dropped
            v = leaves[:, f * Ng:(f + 1) * Ng]
            p_new = v.flat[0]
            assert (v == p_new).all() and abs(p_new - 0.01 ** 0.6) < 1e-6 * p_new
        assert (leaves[:, ring.head * Ng:(ring.head + 1) * Ng] == 0).all()
    assert ring.count_g() == 8 * Ng
    assert_sac_trainers_equal(S, [X for _, X in pairs])
    leaves, totals, beta = S.per_state(n)
    for g, (_, X) in enumerate(pairs):
        l1, t1, b1 = X.per_state(n)
        assert_same(leaves[g], l1, "leaves of trainer %d" % g)
        assert_same(totals[g:g + 1], np.array([t1]), "total of trainer %d" % g)
        assert beta == b1
        assert (l1 != p_new).sum() > (l1 == 0).sum() - Ng            # re-prioritised leaves beyond the empty frame


# ------------------------------------------------------------------ 4. bypass, refusals, launch counts
def test_injected_tape_bypasses_the_trees(env_golden, env27_golden):
    """An injected idx_tape runs the uniform update and leaves the trees untouched: it equals a twin without trees."""
    N, cap = 128, 128 * 6
    (e0, S), = ring_learners(env_golden, env27_golden, N, cap, twins=1)
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=3)
    e1 = make_env(env_golden, env27_golden, N, pool)
    e1.reset(0)
    X = sac(1, seed=7, replay_capacity=cap, lockstep_envs=N)
    X.init_params(1)
    distinct_alphas(X, np.random.default_rng(7))
    engine.sac_train_run(e0, S, 5, do_update=False)
    engine.sac_train_run(e1, X, 5, do_update=False)
    before = S.per_state(S.tree_slots())
    tape = dev(np.random.default_rng(0).choice(S.replay_size(), 64, replace=False).astype(np.int32))
    l0, l1 = torch.zeros(4, device=DEV), torch.zeros(4, device=DEV)
    S.update_replay(tape, losses=l0)
    X.update_replay(tape, losses=l1)
    for role in range(14):
        assert_same(S.get_params(role), X.get_params(role), "role %d" % role)
    assert_same(l0.cpu().numpy(), l1.cpu().numpy(), "losses")
    after = S.per_state(S.tree_slots())
    assert_same(after[0], before[0], "leaves") and after[2] == before[2]


def test_refusals_leave_state_untouched(env_golden, env27_golden):
    S0 = sac(1, lockstep_envs=0)
    with pytest.raises(engine.UavrlError, match="no replay ring"):
        S0.per_enable()
    slots, w = torch.zeros(4, dtype=torch.int32, device=DEV), torch.zeros(4, device=DEV)
    for call in (lambda: S0.per_sample(4), lambda: S0.per_set_errors(slots, w), lambda: S0.per_set_priorities(slots, w.double()),
                 lambda: S0.per_state(4)):
        with pytest.raises(engine.UavrlError, match="prioritised replay not enabled"):
            call()
    s = torch.zeros((8, OBS), device=DEV)
    with pytest.raises(engine.UavrlError, match="bad argument"):         # is_weights is required
        _lib.check(_lib.lib().uavrl_sac_update_batch_per(S0.h, 8, engine._ptr(s), engine._ptr(s[:, :2].contiguous()),
                                                         engine._ptr(w), engine._ptr(s), engine._ptr(w), None, None, None, None,
                                                         None, None))
    assert S0.scalars()["epoch"] == 0
    (env, S), = ring_learners(env_golden, env27_golden, 128, 128 * 6, twins=1)
    with pytest.raises(engine.UavrlError, match="already enabled"):
        S.per_enable()
    engine.sac_train_run(env, S, 3, do_update=False)
    state = S.per_state(S.tree_slots())
    with pytest.raises(engine.UavrlError, match="already enabled"):
        S.per_enable(0.5)
    after = S.per_state(S.tree_slots())
    assert_same(after[0], state[0], "leaves after a refused enable") and after[2] == state[2]
    Y = sac(1, lockstep_envs=1024, replay_capacity=4_300_000)         # 4201 frames x 1024 envs > 4 194 304 slots
    with pytest.raises(engine.UavrlError, match="at most 4194304 slots"):
        Y.per_enable()
    Y.close()


def test_stored_transition_refuses_enable(env_golden, env27_golden):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, 128, max_subgoals=64).make_scenarios(128, seed=3)
    env = make_env(env_golden, env27_golden, 128, pool)
    env.reset(0)
    S = sac(1, lockstep_envs=128, replay_capacity=128 * 6)
    engine.sac_train_run(env, S, 1, do_update=False)
    with pytest.raises(engine.UavrlError, match="before the first transition"):
        S.per_enable()
    with pytest.raises(engine.UavrlError, match="prioritised replay not enabled"):
        S.per_state(4)


@pytest.mark.parametrize("G", [1, 4])
def test_launch_counts(env_golden, env27_golden, G):
    """A lockstep iteration with the trees on: 5 launches without an update (act, env step, the commit's leaf and two level
    refreshes), 17 with one (+ sample, normalise, target, weighted critic, 2 critic steps, actor, actor step, finish, and the
    three write-back launches)."""
    N, B = 128 * G, 64
    (env, S), = ring_learners(env_golden, env27_golden, N, N * 6, twins=1, trainers=G)
    engine.sac_train_run(env, S, 1, do_update=False)
    c0 = _lib.launch_count()
    engine.sac_train_run(env, S, 1, do_update=False)
    assert _lib.launch_count() - c0 == 5
    assert S.replay_size() // G > B
    c0 = _lib.launch_count()
    engine.sac_train_run(env, S, 1)
    assert _lib.launch_count() - c0 == 17


# ------------------------------------------------------------------ 5. data-parallel forms
def test_data_parallel_forms_at_world_one(env_golden, env27_golden):
    """connect_self: update_replay_dp, the split form and sac_train_run_dp each equal update_replay / sac_train_run with the
    trees on, bit for bit, trees included."""
    N, B = 128, 64
    cap = N * 6
    (e0, S), (e1, X) = ring_learners(env_golden, env27_golden, N, cap)
    engine.sac_train_run(e0, S, 4, do_update=False)
    engine.sac_train_run(e1, X, 4, do_update=False)
    S.connect_self()
    for form in ("fused", "split"):
        l0, l1 = torch.zeros(4, device=DEV), torch.zeros(4, device=DEV)
        if form == "fused":
            S.update_replay_dp(B, losses=l0)
        else:
            S.critic_grads(B)
            S.apply_critic_grads()
            S.actor_grads()
            S.apply_actor_grads(l0)
        X.update_replay(losses=l1)
        torch.cuda.synchronize()
        learners_equal(S, X, form, l0, l1)
    engine.sac_train_run_dp(e0, S, 3, B)
    engine.sac_train_run(e1, X, 3)
    learners_equal(S, X, "train_run_dp")


def test_two_simulated_ranks_stay_identical(env_golden, env27_golden):
    """Two ranks on one GPU through the split form (the caller sums the exchange vectors): each rank samples its own trees
    over its own shard, the replicas stay bit-identical and each rank's trees are re-prioritised from its own errors."""
    N, B = 128, 64
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    ranks = []
    for r in range(2):
        pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=10 + r)
        env = make_env(env_golden, env27_golden, N, pool)
        env.reset(0)
        S = sac(1, seed=20 + r, replay_capacity=N * 6, lockstep_envs=N)
        S.init_params(1)
        S.per_enable()
        engine.sac_train_run(env, S, 4, do_update=False)
        ranks.append(S)
    fresh = [S.per_state(S.tree_slots())[0] for S in ranks]
    for _ in range(3):
        for S in ranks:
            S.critic_grads(2 * B)
        tot = ranks[0].exchange_tensor(0) + ranks[1].exchange_tensor(0)
        for S in ranks:
            S.exchange_tensor(0).copy_(tot)
            S.apply_critic_grads()
            S.actor_grads()
        tot = ranks[0].exchange_tensor(1) + ranks[1].exchange_tensor(1)
        for S in ranks:
            S.exchange_tensor(1).copy_(tot)
            S.apply_actor_grads()
    torch.cuda.synchronize()
    for role in range(11):
        assert_same(ranks[0].get_params(role), ranks[1].get_params(role), "replica role %d" % role)
    leaves = [S.per_state(S.tree_slots())[0] for S in ranks]
    for r in range(2):
        assert (leaves[r] != fresh[r]).any()
    assert not np.array_equal(leaves[0], leaves[1])


# ------------------------------------------------------------------ 6. plug-ins
@pytest.mark.parametrize("trainers", ["1", "8"])
def test_env_plugin_trains_on_prioritised_samples(tmp_path, trainers):
    """PathPlan_City_B200 with the SAC XMLs and IsPriority_Replay = 1: an episode trains, every tree holds re-prioritised
    leaves, Is_FL = 1 leaves the trees alone, and save() / Load_Mod round-trip the networks."""
    with env_plugin(tmp_path, IsPriority_Replay="1") as mod:
        env = mod.PathPlan_City_B200(env_dict(*SAC_XML, num_trainers=trainers))
        L = env.Trainer._learner
        info = env.run_eposide(0.3)
        assert info["updates"] > 0 and np.isfinite(info["loss"])
        leaves = L.per_state(L.tree_slots())[0].reshape(L.G, -1)
        for g in range(L.G):
            assert ((np.abs(leaves[g] - 0.01 ** 0.6) > 1e-5) & (leaves[g] != 0)).any(), "trainer %d" % g
        env.Trainer.save()
        env2 = mod.PathPlan_City_B200(env_dict(*SAC_XML, num_trainers=trainers))
        for role in (0, 1, 2):
            assert_same(env2.Trainer._learner.get_params(role), L.get_params(role), "restored role %d" % role)
        env3 = mod.PathPlan_City_B200(env_dict(*SAC_XML, num_trainers=trainers, Is_FL="1", Is_AC="1", FL_Loop="1"))
        L3 = env3.Trainer._learner
        seen = []
        fed = L3.federate_actors

        def spy():
            seen.append(L3.per_state(L3.tree_slots()))
            fed()
            after = L3.per_state(L3.tree_slots())
            assert_same(after[0], seen[-1][0], "leaves across the federation")
        L3.federate_actors = spy
        env3.run_eposide(0.3)
        assert len(seen) == 1


def test_trainer_plugin_refusals_and_weighted_update(tmp_path):
    from uavrl_b200.plugins import xmlconfig
    from uavrl_b200.plugins.SAC_Trainer_B200 import SAC_Trainer_B200
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    param = xmlconfig.XML2Dict(os.path.join(root, "configs", "Trainer_SAC_B200.xml"))["Trainer"]
    param.update(IsPriority_Replay="1", save_loop="0", model_path=str(tmp_path), Batch_Size="16", replay_size="512")
    with pytest.raises(ValueError, match="lockstep ring"):
        SAC_Trainer_B200(dict(param, lockstep_envs="0"))
    tr = SAC_Trainer_B200(dict(param, lockstep_envs="64"))
    L = tr._learner
    rng = np.random.default_rng(1)
    B = 16
    td = dict(states=rng.normal(size=(B, OBS)).astype(np.float32), next_states=rng.normal(size=(B, OBS)).astype(np.float32),
              actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.normal(size=B).astype(np.float32),
              dones=np.zeros(B, np.float32), weights=weights(rng, B))
    n = L.tree_slots()
    slots = rng.choice(n, B, replace=False)
    td["idx"] = slots + n - 1
    # the same weighted update on a twin learner gives the errors written back
    X = engine.SacLearner(OBS, L.cfg.hidden, 2, L.cfg.action_bound, L.cfg.actor_lr, L.cfg.critic_lr, L.cfg.alpha_lr,
                          L.cfg.target_entropy, L.cfg.gamma, L.cfg.tau, batch_size=B, seed=L.cfg.seed)
    for role in range(11):
        X.set_params(role, L.get_params(role))
    ae = torch.zeros(B, device=DEV)
    f = lambda x: dev(np.asarray(x, np.float32))                      # noqa: E731
    X.update_batch_per(f(td["states"]), f(td["actions"]), f(td["rewards"]), f(td["next_states"]), f(td["dones"]), f(td["weights"]), ae)
    tr.update(td)
    leaves = L.per_state(n)[0]
    want = np.minimum(np.abs(ae.cpu().numpy()) + np.float32(0.01), np.float32(1.0)).astype(np.float32) ** np.float32(0.6)
    np.testing.assert_allclose(leaves[slots], want, rtol=1e-6, err_msg="written-back leaves")
    for role in range(3):
        assert_same(L.get_params(role), X.get_params(role), "role %d" % role)
    tr._world = 2
    with pytest.raises(ValueError, match="data-parallel"):
        tr.update(td)
