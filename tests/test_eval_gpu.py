"""Episode records (include/uavrl.h, uavrl_env_set_records) and policy evaluation (uavrl_eval_run, uavrl_sac_eval_run) on one GPU:
every record against what the host accumulates from the per-step outputs, the evaluation against the same suite driven
through the existing calls, bit for bit, the suite's coverage, the absence of side effects on the learner, and the refusals."""
import numpy as np
import pytest
import torch

from gpu_util import MAX_STEP, assert_records_equal, assert_same, compose, dev, learner, sac, short_episode_env, standalone_like
from sac_restatement import actor_fwd, init_state, unpack
from uavrl_b200 import _lib, engine

gpu = pytest.mark.gpu
SHAPE = (100, [64, 64], 27, False)
POWER = dict(P_i=89.0, v_0=4.05, d_0=0.6, rho=1.225, s=0.05, A=0.5, P_b=79.0, F_b=120.0, xi=0.8)     # config/UAV.xml <Fly_power>
FIELDS = list(engine.RECORD_FIELDS)


def make_env(env_golden, env27_golden, n, P, seed=5, auto_reset=False):
    city, params = short_episode_env(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=auto_reset)
    sc = env.make_scenarios(P, seed=seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    return env, sc


def dist(a, b):
    d = a - b
    return np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])


def planner_len(sub, n_sub):
    """CalMod.calculate_path_len of the queue, left to right, in float64"""
    out = 0.0
    for i in range(1, int(n_sub)):
        out = out + float(dist(sub[i - 1], sub[i]))
    return out


def dqn(**kw):
    L = learner(SHAPE, **kw)
    L.init_params(3)
    return L


# ------------------------------------------------------------------ 1. record fields
@gpu
@pytest.mark.parametrize("extras", ["none", "energy", "apf"])
@pytest.mark.parametrize("kind", ["discrete", "continuous"])
def test_record_fields(env_golden, env27_golden, kind, extras):
    """64 envs without auto-reset, one episode each, driven by observe -> act -> step: every record equals what the host reads
    at the ending step (outputs, get_state, get_energy), start2goal and planner_len are the float64 reference formulas."""
    N = 64
    env, sc = make_env(env_golden, env27_golden, N, N, seed=11)
    if extras == "energy":
        env.set_extras(power=POWER)
    elif extras == "apf":
        rng = np.random.default_rng(3)
        nb = env_golden["buildings"].shape[0]
        vel = np.zeros((nb, 3)); vel[:, :2] = rng.normal(0, 1.5, (nb, 2))
        env.set_extras(obstacle_v=vel)
    env.set_records(N)
    env.reset(0)
    L = dqn()
    rng = np.random.default_rng(7)
    steps = np.zeros(N, np.int64); coll = np.zeros(N, np.int64)
    want = {}
    obs = env.observe()
    for t in range(40 * MAX_STEP):
        if kind == "discrete":
            a = L.act(obs, 0.0, is_train=False)
        else:
            a = dev(rng.uniform(-1, 1, N).astype(np.float32))
        out = env.step(a)
        obs = out["obs"]
        ended, info, c = (out[k].cpu().numpy() for k in ("ended", "info", "collision"))
        live = np.array([e not in want for e in range(N)])
        steps[live] += 1; coll[live] += c[live]
        if (ended & live).any():
            st = env.get_state()
            en = env.get_energy() if extras == "energy" else np.zeros(N)
            for e in np.nonzero(ended & live)[0]:
                s = int(st["scenario"][e])
                p = np.array([st["px"][e], st["py"][e], st["pz"][e]])
                want[e] = dict(scenario=s, env=e, ordinal=0, outcome=int(info[e]), steps=int(steps[e]), subgoals=int(st["cursor"][e]),
                               collisions=int(coll[e]), total_score=st["total_score"][e], path_len=st["path_len"][e],
                               start2goal=float(dist(sc["start"][s], sc["goal"][s])), planner_len=planner_len(sc["sub"][s], sc["n_sub"][s]),
                               final_dist=float(dist(p, sc["goal"][s])), energy=en[e])
        if len(want) == N:
            break
    assert len(want) == N, "every env must end its episode"
    rec = env.records()
    assert list(rec["slot"]) == list(range(N))
    for e in range(N):
        for k in FIELDS:
            got = rec[k][e]
            assert np.asarray(got).tobytes() == np.asarray(want[e][k], np.asarray(got).dtype).tobytes(), (e, k, got, want[e][k])
    assert env.records()["slot"].size == 0                       # clear=True emptied them


# ------------------------------------------------------------------ 2. composition
@gpu
@pytest.mark.parametrize("route", ["fp32", "tc"])
def test_eval_equals_composition(env_golden, env27_golden, route):
    N, P, n, first = 64, 300, 150, 290
    L = dqn()
    if route == "fp32":
        L.set_tensor_cores(False)
        assert L.route(N)["tc_fwd"] is None
    else:
        assert L.route(N)["tc_fwd"] is not None
    calls = L.counters()
    E1, _ = make_env(env_golden, env27_golden, N, P)
    res = engine.eval_run(E1, L, n, first_scenario=first)
    assert res["unfinished"] == 0 and res["n_records"] == n
    assert L.counters() == calls
    E2, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
    want = compose(E2, n, first, lambda o: (L.act(o, 0.0, is_train=False), _lib.ACT_DISCRETE27))
    assert_records_equal(res["records"], want, route)
    assert (res["records"]["trainer"] == 0).all()


@gpu
def test_eval_grouped_equals_standalone(env_golden, env27_golden):
    N, P, n, G = 64, 200, 100, 4
    Lg = learner(SHAPE, trainers=G)
    Lg.init_params(5)
    solo = [standalone_like(Lg, SHAPE, g) for g in range(G)]
    E1, _ = make_env(env_golden, env27_golden, N, P)
    res = engine.eval_run(E1, Lg, n, first_scenario=7)
    E2, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
    ng = N // G
    act = lambda o: (torch.cat([solo[g].act(o[g * ng:(g + 1) * ng].contiguous(), 0.0, is_train=False) for g in range(G)]),  # noqa: E731
                     _lib.ACT_DISCRETE27)
    assert_records_equal(res["records"], compose(E2, n, 7, act), "grouped")
    assert list(res["records"]["trainer"]) == list((np.arange(n) % N) // ng)


@gpu
def test_sac_mean_eval_equals_composition(env_golden, env27_golden):
    N, P, n = 64, 200, 96
    S = sac(trainers=2)
    S.init_params(4)
    E1, _ = make_env(env_golden, env27_golden, N, P)
    res = engine.sac_eval_run(E1, S, n, first_scenario=3, mean_action=True)
    assert res["unfinished"] == 0
    E2, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
    want = compose(E2, n, 3, lambda o: (S.act(o, mean=True), _lib.ACT_CONT_F32X2))
    assert_records_equal(res["records"], want, "sac mean")


@gpu
def test_mean_action_vs_float64():
    obs, hid, bound = 100, 64, 1.0
    rng = np.random.default_rng(9)
    st = init_state(rng, obs, hid)
    S = engine.SacLearner(obs, hid, 2, bound, seed=1)
    S.set_params(0, st["actor"])
    P = unpack(st["actor"], "actor", obs, hid)
    s = rng.normal(0, 1, (1000, obs)).astype(np.float32)
    f = actor_fwd(P, s.astype(np.float64), np.zeros((1000, 2)), bound)
    got = S.act(dev(s), mean=True).cpu().numpy().astype(np.float64)
    (_, _), (Wm, bm), _ = P
    scale = f["h"] @ np.abs(Wm).T + np.abs(bm)
    near = (np.abs(f["z"]) <= 5e-5 * f["zabs"]).any(1)
    err = np.abs(got - f["act"])[~near] - bound * (1e-6 + 2e-5 * scale[~near])
    assert (err <= 0).all(), float(err.max())
    assert S.scalars()["epoch"] == 0


# ------------------------------------------------------------------ 3. suite coverage
@gpu
@pytest.mark.parametrize("n,first", [(150, 0), (40, 5), (64, 290), (0, 0)], ids=["n_not_multiple", "n_lt_N", "wrap", "empty"])
def test_suite_coverage(env_golden, env27_golden, n, first):
    N, P = 64, 300
    L = dqn()
    env, _ = make_env(env_golden, env27_golden, N, P)
    env.reset(11)
    env.step(L.act(env.observe(), 0.0, is_train=False))
    before = env.get_state()
    res = engine.eval_run(env, L, n, first_scenario=first)
    r = res["records"]
    assert res["unfinished"] == 0 and res["n_records"] == n
    assert list(r["scenario"]) == [(first + k) % P for k in range(n)]
    assert list(r["env"]) == [k % N for k in range(n)] and list(r["ordinal"]) == [k // N for k in range(n)]
    assert ((r["outcome"] == 1) | (r["outcome"] == 2)).all()
    after = env.get_state()
    for k in before:
        assert_same(after[k][n:], before[k][n:], "parked env state " + k)
    if n == 0:
        assert res["iterations"] == 0


@gpu
def test_max_iters_cut(env_golden, env27_golden):
    L = dqn()
    env, _ = make_env(env_golden, env27_golden, 64, 300)
    res = engine.eval_run(env, L, 300, max_iters=5)
    assert res["iterations"] == 5 and res["unfinished"] > 0
    assert res["n_records"] + res["unfinished"] == 300
    assert (res["records"]["outcome"] != 0).sum() == res["n_records"]


# ------------------------------------------------------------------ 4. no side effects
def dqn_pair_state(L, N, capacity):
    slots = (capacity // N + 1) * N                              # ring frames x envs: the tree's leaves
    return [L.get_params(w) for w in range(4)] + [np.array(L.counters())] + list(L.gather(np.arange(L.replay_size()))) + \
        [np.atleast_1d(x) for x in L.per_state(slots)]


@gpu
def test_eval_between_train_chunks_changes_nothing(env_golden, env27_golden):
    N, P = 64, 200
    outs = []
    for with_eval in (False, True):
        L = learner(SHAPE, lockstep_envs=N, replay_capacity=4096, batch_size=32)
        L.init_params(2)
        L.per_enable()
        env, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
        env.reset(0)
        s1 = engine.train_run(env, L, 40, 0.3)
        if with_eval:
            ev, _ = make_env(env_golden, env27_golden, N, P, seed=6)
            engine.eval_run(ev, L, 100)
        s2 = engine.train_run(env, L, 40, 0.3)
        outs.append((dqn_pair_state(L, N, 4096), [s.env_steps for s in (s1, s2)] + [s.episodes_ended for s in (s1, s2)], env.get_state()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert_same(a, b, "learner state")
    assert outs[0][1] == outs[1][1]
    for k in outs[0][2]:
        assert_same(outs[0][2][k], outs[1][2][k], "training env " + k)


@gpu
def test_sac_sampled_eval_changes_nothing_and_repeats(env_golden, env27_golden):
    N, P = 64, 200
    outs, recs = [], []
    for with_eval in (False, True):
        S = sac(trainers=2, lockstep_envs=N, replay_capacity=4096)
        S.init_params(2)
        S.per_enable()
        env, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
        env.reset(0)
        engine.sac_train_run(env, S, 40)
        if with_eval:
            ev, _ = make_env(env_golden, env27_golden, N, P, seed=6)
            recs = [engine.sac_eval_run(ev, S, 100, first_scenario=4)["records"] for _ in range(2)]
        engine.sac_train_run(env, S, 40)
        outs.append([S.get_params(r) for r in range(11)] + [S.alpha(), np.array(list(S.scalars().values()))] +
                    list(S.gather(np.arange(S.replay_size()))) + [np.atleast_1d(x) for x in S.per_state(S.tree_slots())])
    for a, b in zip(*outs):
        assert_same(a, b, "sac learner state")
    assert_records_equal(recs[0], recs[1], "sampled evaluation repeated")


@gpu
def test_records_in_training_loop(env_golden, env27_golden):
    N, P = 64, 200
    outs = []
    for on in (False, True):
        L = learner(SHAPE, lockstep_envs=N, replay_capacity=4096, batch_size=32)
        L.init_params(2)
        env, _ = make_env(env_golden, env27_golden, N, P, auto_reset=True)
        if on:
            env.set_records(100000)
        env.reset(0)
        st = engine.train_run(env, L, 80, 0.3)
        outs.append(([L.get_params(w) for w in range(4)], (st.env_steps, st.episodes_ended, st.collisions, st.n_success, st.n_lose)))
        if on:
            rec = env.records()
            assert rec["slot"].size == st.episodes_ended > 0 and rec["n_dropped"] == 0
            # n_success also counts the steps that pop an intermediate sub-goal; every 'lose' step ends an episode
            assert (rec["outcome"] == 2).sum() == st.n_lose and (rec["outcome"] == 1).sum() == st.episodes_ended - st.n_lose
    for a, b in zip(outs[0][0], outs[1][0]):
        assert_same(a, b, "parameters with records on")
    assert outs[0][1] == outs[1][1]


# ------------------------------------------------------------------ 5. refusals
@gpu
def test_refusals_leave_state(env_golden, env27_golden):
    N, P = 64, 100
    L = dqn()
    env, _ = make_env(env_golden, env27_golden, N, P)
    env.reset(0)
    before, params = env.get_state(), L.get_params(0)

    def refused(fn, match):
        with pytest.raises(engine.UavrlError, match=match):
            fn()
        after = env.get_state()
        for k in before:
            assert_same(after[k], before[k], "env state after a refusal: " + k)
        assert_same(L.get_params(0), params, "learner after a refusal")

    refused(lambda: engine.eval_run(env, L, -1), "n_episodes")
    city, params_u = short_episode_env(env_golden, env27_golden)
    bare = engine.EnvBatch(city, params_u, N, max_subgoals=64)
    with pytest.raises(engine.UavrlError, match="set_pool"):
        engine.eval_run(bare, L, 4)
    L64 = engine.Learner(64, [32], 27, seed=1)
    refused(lambda: engine.eval_run(env, L64, 4), "100 wide")
    L5 = engine.Learner(100, [32], 5, seed=1)
    refused(lambda: engine.eval_run(env, L5, 4), "27 actions")
    env6, _ = make_env(env_golden, env27_golden, 6, P)
    with pytest.raises(engine.UavrlError, match="multiple of the trainer count"):
        engine.eval_run(env6, learner(SHAPE, trainers=4), 4)
    S = sac()
    with pytest.raises(engine.UavrlError, match="mean_action"):
        _lib.check(_lib.lib().uavrl_sac_eval_run(env.h, S.h, 0, 4, 2, 0, None, None, None))
    if torch.cuda.device_count() > 1:
        L1 = learner(SHAPE, device=1)
        refused(lambda: engine.eval_run(env, L1, 4), "different devices")


# ------------------------------------------------------------------ 6. plug-in
@gpu
@pytest.mark.parametrize("trainer,agent,extra", [("Trainer_DDQN_B200.xml", "UAV_energy_B200.xml", {}),
                                                 ("Trainer_SAC_B200.xml", "UAV_continuous_B200.xml", {"Is_AC": "1"})], ids=["ddqn", "sac"])
def test_plugin_run_evaluation(tmp_path, trainer, agent, extra):
    """run_evaluation after run_eposide leaves the training env and the trainer as they were, grows Testing_time and writes
    one CSV row per episode; record_episodes = 1 adds generate_train_result's fields to run_eposide's result."""
    import csv
    import os
    from gpu_util import env_dict, env_plugin
    ed = env_dict(trainer, agent, record_episodes="1", eval_episodes="40", eval_envs="16", **extra)
    with env_plugin(tmp_path / "Mod") as mod:
        cwd = os.getcwd()
        os.chdir(tmp_path)
        try:
            env = mod.PathPlan_City_B200(ed)
            info = env.run_eposide(0.3)
            L = env.Trainer._learner
            if isinstance(L, engine.SacLearner):
                snap = lambda: [L.get_params(r) for r in range(11)] + [L.alpha()]  # noqa: E731
            else:
                snap = lambda: [L.get_params(w) for w in range(4)] + [np.array(L.counters())]  # noqa: E731
            before, state, t0 = snap(), env.batch.get_state(), env.Agents[0].Testing_time
            out = env.run_evaluation()
        finally:
            os.chdir(cwd)
    assert {"path_len", "start2goal", "len_Astar", "ReachGoal"} <= set(info) and info["len_Astar"] > 0
    for a, b in zip(before, snap()):
        assert_same(a, b, "trainer after run_evaluation")
    after = env.batch.get_state()
    for k in state:
        assert_same(after[k], state[k], "training env after run_evaluation: " + k)
    assert env.Agents[0].Testing_time > t0
    assert out["episodes"] + out["unfinished"] == 40 and out["success"] + out["lose"] == out["episodes"]
    assert len(out["success_rate_per_trainer"]) == 8
    rows = list(csv.reader(open(os.path.join(tmp_path, out["csv"]))))
    assert len(rows) == 1 + out["episodes"] and rows[0][0] == "position"
