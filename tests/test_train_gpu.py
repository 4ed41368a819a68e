"""The fused lockstep loop (uavrl_train_run): what it stores in the replay ring must be exactly what
the reference's run_thread_OffPolicy stores (state, action, reward, next_state, returned done), checked
by replaying the stored actions through the CPU oracle."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import assert_obs, city_and_params

pytestmark = pytest.mark.gpu


def test_lockstep_ring_matches_oracle_rollout(env_golden, env27_golden):
    from uavrl_b200 import engine
    city, params, ocity, oparams = city_and_params(env_golden, env27_golden)
    N, T, K = 96, 40, 64                       # N not a multiple of 32: ragged last CTA
    env = engine.EnvBatch(city, params, N, max_subgoals=K, auto_reset=False)
    sc = env.make_scenarios(N, seed=4)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=N * (T + 5),
                       lockstep_envs=N, seed=3)
    L.init_params(0)
    st = engine.train_run(env, L, T, eps=0.7, do_update=False)
    assert st.env_steps == N * T and st.updates == 0
    assert L.replay_size() == N * T
    s, a, r, s2, d = L.gather(np.arange(N * T))
    s = s.reshape(T, N, 100); s2 = s2.reshape(T, N, 100)
    a = a.reshape(T, N); r = r.reshape(T, N); d = d.reshape(T, N)
    ob = O.OracleBatch(ocity, oparams, N, K)
    ob.reset(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    obs = ob.state(want64=True)[1]
    net = O.make_net(100, [64, 64], 27, 0)
    p = L.get_params(0)
    n_greedy = 0
    for t in range(T):
        assert_obs(s[t], obs, "s t%d" % t)
        assert a[t].min() >= 0 and a[t].max() < 27
        n_greedy += int((a[t] == O.net_forward(net, p, s[t]).argmax(1)).sum())
        rew, done, info, coll, _ = ob.step_(a[t].astype(np.float64), O.ACT_DISCRETE27, want_obs=False)
        obs = ob.state(want64=True)[1]
        np.testing.assert_allclose(r[t], rew, rtol=1e-5, atol=1e-5)
        assert np.array_equal(d[t], done)
        assert_obs(s2[t], obs, "s2 t%d" % t)
    frac = n_greedy / (N * T)
    assert 0.25 < frac < 0.45                  # (1 - eps) + eps/27 = 0.326
    env.close(); L.close()


def test_training_loop_learns_and_counts(env_golden, env27_golden):
    from uavrl_b200 import engine
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N = 512
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(1024, seed=8)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=N, replay_capacity=N * 64,
                       lockstep_envs=N, seed=1, update_loop=3)
    L.init_params(1)
    p0 = L.get_params(0)
    st = engine.train_run(env, L, 200, eps=0.1)
    assert st.env_steps == N * 200
    assert st.updates == 199                    # the first iteration leaves exactly Batch_Size transitions: not > Batch_Size
    assert L.counters() == (200, 199)
    assert np.isfinite(st.last_loss) and np.isfinite(st.sum_reward)
    assert st.episodes_ended > 0
    p1 = L.get_params(0)
    assert np.isfinite(p1).all() and np.abs(p1 - p0).max() > 1e-3
    # ring wrapped (200 iterations through 65 frames) and stayed consistent
    assert L.replay_size() == N * 64
    env.close(); L.close()


@pytest.mark.parametrize("algo", ["dqn", "ddqn"])
def test_dependent_launch_overlap_changes_nothing(env_golden, env27_golden, algo):
    """Programmatic dependent launch inside the loop (kernel k+1's prologue overlaps kernel k's tail,
    uavrl_set_pdl) and the TD-target pass folded into the training kernel (uavrl_set_fuse_td) are scheduling changes only:
    150 lockstep iterations with every on/off combination end in bit-identical parameters, replay contents, env state
    and counters."""
    from uavrl_b200 import _lib, engine
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N = 1024
    out = []
    try:
        for pdl, fuse_td in ((1, 1), (0, 0), (1, 0), (0, 1)):
            _lib.lib().uavrl_set_pdl(pdl)
            _lib.lib().uavrl_set_fuse_td(fuse_td)
            env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
            sc = env.make_scenarios(1024, seed=8)
            env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
            env.reset(0)
            L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DQN if algo == "dqn" else engine.ALGO_DDQN,
                               batch_size=N, replay_capacity=N * 32, lockstep_envs=N, seed=1, update_loop=3)
            L.init_params(0)
            engine.train_run(env, L, 8, eps=1.0, do_update=False)            # collection-only chain: act -> env -> act
            st = engine.train_run(env, L, 150, eps=0.2)
            torch.cuda.synchronize()
            s, a, r, s2, d = L.gather(np.arange(L.replay_size()))
            es = env.get_state()
            out.append(dict(p=L.get_params(0), t=L.get_params(1), s=s, a=a, r=r, d=d, px=es["px"], step=es["step"],
                            stats=(st.env_steps, st.updates, st.episodes_ended, st.collisions, st.n_success, st.n_lose,
                                   st.sum_reward, st.last_loss)))
            env.close(); L.close()
    finally:
        _lib.lib().uavrl_set_pdl(1)                 # library defaults: PDL on, fused TD on
        _lib.lib().uavrl_set_fuse_td(1)
    a = out[0]
    for b in out[1:]:
        assert a["stats"][:6] == b["stats"][:6] and a["stats"][1] == 150 and a["stats"][7] == b["stats"][7]
        assert abs(a["stats"][6] - b["stats"][6]) <= 1e-9 * abs(b["stats"][6])       # sum_reward: fp64 atomics, order-dependent
        for k in ("p", "t", "s", "a", "r", "d", "px", "step"):
            assert np.array_equal(a[k], b[k]), k


def test_fused_td_on_64_row_tiles_changes_nothing(env_golden, env27_golden):
    """Batches between 4 737 and 9 472 samples (BASELINE configs[3]: 8 192 per GPU) train on 64-row tiles, one per CTA, with the
    TD-target passes inside the training kernel; 40 double-DQN iterations end in the same bits as with stand-alone TD passes."""
    from uavrl_b200 import _lib, engine
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N = 6144
    out = []
    try:
        for fuse_td in (1, 0):
            _lib.lib().uavrl_set_fuse_td(fuse_td)
            env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
            sc = env.make_scenarios(1024, seed=8)
            env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
            env.reset(0)
            L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=N, replay_capacity=N * 8, lockstep_envs=N, seed=1,
                               update_loop=3)
            L.init_params(0)
            assert L.td_fused() == bool(fuse_td)
            engine.train_run(env, L, 3, eps=1.0, do_update=False)
            st = engine.train_run(env, L, 40, eps=0.2)
            torch.cuda.synchronize()
            out.append(dict(p=L.get_params(0), t=L.get_params(1), loss=st.last_loss, updates=st.updates))
            env.close(); L.close()
    finally:
        _lib.lib().uavrl_set_fuse_td(1)
    a, b = out
    assert a["updates"] == b["updates"] == 40 and np.isfinite(a["p"]).all()
    assert np.array_equal(a["p"], b["p"]) and np.array_equal(a["t"], b["t"]) and a["loss"] == b["loss"]
