"""The host-driven plug-in loop (PathPlan_City_B200.run_step_OffPolicy with host_driven = 1: states -> Trainer.get_action ->
Move_Agents -> replay_memory.add_batch -> Trainer.learn_off_policy, host arrays at every boundary) and the paired replay store it
trains from (lockstep_envs = 0), checked against independent statements of each part:

- the store and the learner's schedule restated on the host (replay_restatement.Paired / PairedLoop): every update() draws
  sample(seed, epoch, count, B) from the rows a host copy of the pushes holds at those logical indices, bit for bit, at every
  route of the Q-network, and equals float64 at the shipped networks;
- get_action from host arrays: the restated eps-greedy draw and the float64 argmax, one act call per get_action;
- run_step_OffPolicy: the env step against the CPU oracle on the same scenario pool, the stored transitions against what the
  step returned, the updates against a twin learner fed explicit batches and against float64;
- the e2e workload as the benchmark builds it, against the same loop composed by hand from engine objects;
- prioritised replay through the trainer's replay facade after the store wraps, against the oracle's SumTree.

Bounds, exemptions and the tally of kink / tie rows are those of test_ring_updates_gpu.py (qnet_restatement.py)."""
import collections
import importlib
import os

import numpy as np
import pytest
import torch

import oracle as O
import replay_restatement as R
from gpu_util import ROOT, assert_close64, assert_obs, dev, env_dict, env_plugin
from qnet_restatement import (Tally, abs_err_bound, big_inputs, check_actions, f64_forward, f64_unpack, f64_update, net_layers,
                              tie_allowance, trunk_exempt)
from shapes import ROUTES, SHIPPED, net_id, shape_id
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu

LR, GAMMA = 5e-4, 0.99                 # the shipped Trainer XMLs' LEARNING_RATE and gamma
F64 = ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len")
XMLS = {"dqn": "Trainer_DQN_B200.xml", "ddqn": "Trainer_DDQN_B200.xml", "dueling": "Trainer_DuelingDQN_B200.xml"}


# ------------------------------------------------------------------ helpers
class Mirror:
    """Host copy of a paired store: the rows of every push in the slots Paired assigns them."""

    def __init__(self, cap, in_dim):
        self.P = R.Paired(cap)
        self.s = np.zeros((cap, in_dim), np.float32); self.s2 = np.zeros((cap, in_dim), np.float32)
        self.a = np.zeros(cap, np.int32); self.r = np.zeros(cap, np.float32); self.d = np.zeros(cap, np.uint8)

    def push(self, s, a, r, s2, d):
        slots = self.P.push(len(a))
        self.s[slots], self.a[slots], self.r[slots], self.s2[slots], self.d[slots] = s, a, r, s2, d
        return slots

    def rows(self, j):
        sl = self.P.slot(j)
        return self.s[sl], self.a[sl], self.r[sl], self.s2[sl], self.d[sl]


def same_rows(got, want, what):
    for k, (x, y) in enumerate(zip(got, want)):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), (what, "sa r s2 d"[k])


def shape_of(L):
    return (L.in_dim, L.hidden, L.n_actions, L.dueling)


def twin_of(L):
    """A learner without a store in L's state (parameters, target, Adam moments, counters, tensor-core setting)."""
    c = L.cfg
    X = engine.Learner(L.in_dim, L.hidden, L.n_actions, L.dueling, c.algo, lr=c.lr, gamma=c.gamma, batch_size=c.batch_size,
                       update_loop=c.update_loop, replay_capacity=max(1000, 2 * c.batch_size), seed=c.seed)
    X.set_tensor_cores(bool(L.route(c.batch_size)["tc_fwd"]))
    assert X.route(c.batch_size) == L.route(c.batch_size)
    for w in range(4):
        X.set_params(L.get_params(w), w)
    X.set_counters(*L.counters())
    return X


def explicit_update(X, batch):
    s, a, r, s2, d = batch
    loss = torch.zeros(1, device="cuda")
    X.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), loss)
    return loss


def follow(X, u, batch):
    """The twin's half of one update() / learn_off_policy: an explicit update on the restated rows, or the epoch alone."""
    if u is None:
        e, t = X.counters()
        X.set_counters(e + 1, t)
        return None
    return explicit_update(X, batch)


def assert_twins(L, X, loss, xloss, what):
    torch.cuda.synchronize()
    assert L.counters() == X.counters(), (what, L.counters(), X.counters())
    for w in range(4):
        assert np.array_equal(L.get_params(w), X.get_params(w)), (what, w)
    if xloss is not None:
        assert np.array_equal(np.float32(float(loss)), np.float32(float(xloss))), (what, float(loss), float(xloss))


def judge_update(L, before, ctr, batch, epoch, hard, loss, tally):
    """L's last update, made from the vectors `before` and counters ctr on the rows `batch` at `epoch`, against the float64
    update (loss, gradient) and the oracle's Adam chain (parameters, target): the bounds of test_ring_updates_gpu.py, plus
    1e-5 of the magnitudes a gradient entry sums (f64_update's abs_terms).  The long host-driven runs store 'lose' rewards,
    whose TD errors make an entry's products cancel far below their own size; fp32-grade sums keep an error of that size.
    Entries where that term decides get the parameter allowance of the other uncertain entries."""
    in_dim, hidden, n_actions, dueling = shape_of(L)
    algo = L.cfg.algo
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    s, a, r, s2, d = batch
    d = d.astype(np.float32)
    B = s.shape[0]
    l64, g64, _, _, mag = f64_update(layers, algo, dueling, before[0], before[1], s, a, r, s2, d, gamma=GAMMA, abs_terms=True)
    kmask, krows = trunk_exempt(layers, len(hidden), f64_unpack(layers, before[0]), dueling, s)
    lal, gal, trows = tie_allowance(layers, algo, dueling, before[0], before[1], (s, a, r, s2, d), L.P, gamma=GAMMA)
    tally.rows += B; tally.kink_rows += krows; tally.tie_rows += trows
    tally.entries += L.P; tally.exempt += int((kmask | (gal > 0)).sum())
    cancel = 1e-5 * mag > 2e-4 * np.abs(g64) + 2e-5
    tally.exempt += int(cancel.sum())
    gg = L.get_params(4).astype(np.float64)
    err = np.abs(gg - g64) - (2e-4 * np.abs(g64) + 2e-5 + gal + 1e-5 * mag)
    err[kmask] = 0
    k = int(err.argmax())
    assert (err <= 0).all(), (epoch, float(err.max()), k, gg[k], g64[k], mag[k])
    assert abs(loss - l64) <= 2e-5 * abs(l64) + lal, (epoch, loss, l64)
    OL = O.OracleLearner(O.make_net(in_dim, hidden, n_actions, int(dueling)), algo, before[0], gamma=GAMMA, lr=LR, update_loop=3)
    OL.target[:] = before[1]; OL.m[:] = before[2]; OL.v[:] = before[3]; OL.t.value = ctr[1]
    OL.epoch = epoch - 1
    lo, _ = OL.update(s, a, r, s2, d)
    assert abs(lo - l64) <= 2e-5 * abs(l64) + lal, (epoch, lo, l64)
    allow = np.where(kmask | (gal > 0) | cancel | ((np.abs(g64) < 1e-5) & (g64 != 0)), 4 * LR, 2e-5)
    local, target = L.get_params(0), L.get_params(1)
    for got, want in ((local, OL.local), (target, OL.target)):
        dp = np.abs(got - want)
        assert (dp <= allow).all(), (epoch, float(dp.max()), int(dp.argmax()))
    # the hard target update lands exactly on the epochs the schedule names
    assert np.array_equal(target, local) if hard else np.array_equal(target, before[1]), (epoch, hard)


def random_rows(rng, n, in_dim, n_actions):
    return (rng.normal(0, 1, (n, in_dim)).astype(np.float32), rng.integers(0, n_actions, n).astype(np.int32),
            rng.normal(0, 1, n).astype(np.float32), rng.normal(0, 1, (n, in_dim)).astype(np.float32),
            (rng.random(n) < 0.1).astype(np.uint8))


def obs_rows(g, rng, n, n_actions):
    """Transitions whose states are golden observations plus noise (the scales the learner sees)."""
    return (big_inputs(g, n, rng), rng.integers(0, n_actions, n).astype(np.int32), rng.normal(0, 1, n).astype(np.float32),
            big_inputs(g, n, rng), (rng.random(n) < 0.1).astype(np.uint8))


def store_state(P, B, n):
    """Which of the paired store's states the push of n transitions left."""
    if P.count <= B:
        return "count<=B"
    if P.count == B + 1:
        return "B+1"
    if P.count < P.slots:
        return "not_full"
    return "full" if P.head == 0 and n != P.slots else "wrapped"


# ------------------------------------------------------------------ (a) sampled updates from the paired store, bit for bit
# capacity 150, B = 64: 30 and 64 (= B, skipped), 65 (= B + 1, the first draw), 115, 150 (exactly full), then wrapped once on
# a ragged boundary (head 47), a push of exactly the capacity, and three more wraps' worth of ragged pushes
PUSHES_A = (30, 34, 1, 50, 35, 47, 150, 120, 97, 13)


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "fp32"])
@pytest.mark.parametrize("shape", ROUTES, ids=shape_id)
def test_paired_update_samples_restated_indices(shape, tc):
    """update() without a tape equals update_batch on the rows a host copy of the pushes holds at the restated indices, bit for
    bit (parameters, target, Adam moments, loss, counters), after every push; a call at count <= B advances the epoch only."""
    in_dim, hidden, n_actions, dueling, route = shape
    cap, B, seed = 150, 64, 11
    L = engine.Learner(in_dim, hidden, n_actions, bool(dueling), engine.ALGO_DDQN, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3,
                       replay_capacity=cap, seed=seed)
    L.init_params(4)
    assert L.set_tensor_cores(tc) == (tc and route[0] is not None)
    X = twin_of(L)
    M = Mirror(cap, in_dim)
    loop = R.PairedLoop(M.P, seed, B, update_loop=3)
    rng = np.random.default_rng(in_dim + 1000 * len(hidden))
    seen = collections.Counter()
    for n in PUSHES_A:
        batch = random_rows(rng, n, in_dim, n_actions)
        L.push(*map(dev, batch))
        M.push(*batch)
        assert L.replay_size() == M.P.count
        same_rows(L.gather(M.P.newest(n)), batch, ("push", n))
        loss = torch.zeros(1, device="cuda")
        L.update(loss=loss)
        u = loop.update()
        xl = follow(X, u, None if u is None else M.rows(u[1]))
        assert_twins(L, X, loss, xl, (n, M.P.count, M.P.head))
        assert L.counters() == (loop.epoch, loop.adam_t)
        seen[store_state(M.P, B, n)] += 1
    assert seen["count<=B"] == 2 and seen["B+1"] == 1 and seen["full"] == 1 and seen["wrapped"] == 5, seen
    assert loop.adam_t == 8 and loop.epoch == 10
    L.close(); X.close()


# ------------------------------------------------------------------ (b) the same updates against float64
F64_LEGS = [(net, algo) for net in SHIPPED for algo in ((engine.ALGO_DUELING,) if net[3] else (engine.ALGO_DQN, engine.ALGO_DDQN))]
ALGO_NAME = {engine.ALGO_DQN: "dqn", engine.ALGO_DDQN: "ddqn", engine.ALGO_DUELING: "dueling"}


def paired_pushes(B):
    """capacity and pushes for batch B: two pushes up to B (skipped), B + 1, exactly full, wrapped on a ragged boundary, a push
    of exactly the capacity, wrapped again."""
    cap = 2 * B + B // 2 + 3
    return cap, [B // 2, B - B // 2, 1, cap - B - 1, cap // 3 + 5, cap, 2 * cap // 3 + 1]


@pytest.mark.parametrize("B", [64, 4096])
@pytest.mark.parametrize("net,algo", F64_LEGS, ids=["%s-%s" % (net_id(n), ALGO_NAME[a]) for n, a in F64_LEGS])
def test_paired_updates_vs_float64(dqn_golden, net, algo, B):
    """The shipped networks under their trainers: every update() the paired store samples (B = 64: 32-row training tiles;
    B = 4096, the e2e batch: 64-row tiles) equals float64 on the restated rows; skipped calls leave every vector unchanged."""
    in_dim, hidden, n_actions, dueling = net
    shape = (in_dim, hidden, n_actions, bool(dueling))
    cap, pushes = paired_pushes(B)
    seed = 5
    L = engine.Learner(*shape, algo, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3, replay_capacity=cap, seed=seed)
    L.init_params(6)
    M = Mirror(cap, in_dim)
    loop = R.PairedLoop(M.P, seed, B, update_loop=3)
    rng = np.random.default_rng(B + algo)
    tally = Tally()
    n_up = n_hard = 0
    for n in pushes:
        batch = obs_rows(dqn_golden, rng, n, n_actions)
        L.push(*map(dev, batch))
        M.push(*batch)
        before = [L.get_params(w) for w in range(4)]
        ctr = L.counters()
        loss = torch.zeros(1, device="cuda")
        L.update(loss=loss)
        u = loop.update()
        torch.cuda.synchronize()
        assert L.counters() == (loop.epoch, loop.adam_t)
        if u is None:
            for w in range(4):
                assert np.array_equal(L.get_params(w), before[w]), (n, w)
            continue
        epoch, idx, hard = u
        judge_update(L, before, ctr, M.rows(idx), epoch, hard, float(loss), tally)
        n_up += 1; n_hard += hard
    tally.check()
    assert n_up == len(pushes) - 2 and n_hard >= 1 and M.P.count == cap
    L.close()


# ------------------------------------------------------------------ (c) get_action from host arrays
def trainer_plugin(tmp_path, xml, **over):
    """A trainer plug-in built from configs/<xml> the way the env plug-in builds it, no periodic save, checkpoints under
    tmp_path; `over` overrides Trainer XML entries (strings)."""
    from uavrl_b200.plugins import xmlconfig
    tdict = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", xml))["Trainer"]
    tdict.update(dict(name="UAV_0", Batch_Size="64", replay_size="1000", save_loop="0", model_path=str(tmp_path)), **over)
    ttype = tdict["Trainer_Type"]
    return getattr(importlib.import_module("uavrl_b200.plugins." + ttype), ttype)(tdict)


@pytest.mark.parametrize("is_train", [1, 0], ids=["train", "eval"])
def test_get_action_from_host_arrays(dqn_golden, tmp_path, is_train):
    """Trainer.get_action on host rows: the restated eps-greedy draw of act call k on the k-th call, the float64 argmax on
    greedy rows; the single-state form returns a Python int; Is_Train = 0 is greedy whatever eps is."""
    tr = trainer_plugin(tmp_path, "Trainer_DQN_B200.xml", Is_Train=str(is_train))
    L = tr._learner
    rng = np.random.default_rng(3 + is_train)
    call = 0
    for N in (1, 31, 257, 4096):
        for eps in (0.0, 0.3, 1.0):
            s = big_inputs(dqn_golden, N, rng)
            p = L.get_params(0)
            out = tr.get_action(s[0] if N == 1 else s, eps)
            if N == 1:
                assert type(out) is int
                a = np.array([out], np.int32)
            else:
                assert isinstance(out, np.ndarray) and out.dtype == np.int32 and out.shape == (N,)
                a = out.copy()
            check_actions(s, a, L.cfg.seed, call, p[None], eps if is_train else 0.0, shape_of(L))
            call += 1
    L.close()


# ------------------------------------------------------------------ (d) run_step_OffPolicy against a restated host loop
def host_env(tmp_path, algo, N, cap, B=64):
    """The env plug-in from configs/PathPlan_City_B200.xml with host_driven = 1, N UAVs, a pool of 2 N scenarios and the
    trainer of configs/<XMLS[algo]> at batch B and replay_size cap."""
    with env_plugin(tmp_path, Batch_Size=str(B), replay_size=str(cap)) as mod:
        return mod.PathPlan_City_B200(env_dict(XMLS[algo], num_UAV=str(N), num_trainers="1", host_driven="1", scenario_pool=str(2 * N)))


class OracleEnv:
    """The CPU oracle's batch on the plug-in's scenario pool, with the in-kernel restart (an ended UAV restarts from scenario
    (scen + N) mod P)."""

    def __init__(self, env):
        b = env.batch
        self.ocity = O.OracleCity(env.len, env.width, env.h, env.buildings_table)
        u = env.uav_params
        self.oparams = O.UavParams(u.max_v, u.min_v, u.steering, u.climb_rate, u.max_step)
        self.sc = sc = b.make_scenarios(env.pool_size, seed=42, rrt_step=env.sub_granularity)
        pool = b.get_pool()
        for k in ("start", "goal", "sub", "n_sub"):
            assert np.array_equal(pool[k], sc[k]), k
        self.N, self.P, self.K = env.num_UAV, env.pool_size, b.K
        self.scen = np.arange(self.N) % self.P                  # Scene_Random_Reset at construction: reset(0)
        self.ob = O.OracleBatch(self.ocity, self.oparams, self.N, self.K)
        self.ob.reset(*(sc[k][self.scen] for k in ("start", "goal", "heading", "sub", "n_sub")))
        self.restarts = 0

    def step(self, a):
        rew, done, info, coll, _ = self.ob.step_(a.astype(np.float64), O.ACT_DISCRETE27, want_obs=False)
        ob, sc = self.ob, self.sc
        ended = np.nonzero(ob.done)[0]
        if ended.size:
            self.scen[ended] = (self.scen[ended] + self.N) % self.P
            s = self.scen[ended]
            fresh = O.OracleBatch(self.ocity, self.oparams, ended.size, self.K)
            fresh.reset(sc["start"][s], sc["goal"][s], sc["heading"][s], sc["sub"][s], sc["n_sub"][s])
            for k in F64 + ("step", "cursor", "n_sub", "done", "alias0"):
                getattr(ob, k)[ended] = getattr(fresh, k)
            ob.goal[ended] = fresh.goal; ob.sub[ended] = fresh.sub
            self.restarts += ended.size
        return rew, done, info

    def check(self, env, s2, r, d, info, want, what):
        rew, done, info_o = want
        assert np.array_equal(d.view(np.uint8), done) and np.array_equal(info, info_o), what
        np.testing.assert_allclose(r, rew, rtol=1e-5, atol=1e-5, err_msg=str(what))
        st = env.batch.get_state()
        assert np.array_equal(st["scenario"], self.scen), what
        assert np.array_equal(st["step"], self.ob.step) and np.array_equal(st["cursor"], self.ob.cursor), what
        assert np.array_equal(st["done"], self.ob.done), what
        assert_close64(st["reward64"], rew, 1e-9, ("reward64",) + what)
        for k in F64:
            assert_close64(st[k], getattr(self.ob, k), 1e-9, (k,) + what)
        assert_obs(s2, self.ob.state(want64=True)[1], str(what))


def age_episodes(env, rng, oe=None):
    """Step counters of every UAV moved to 50-1 steps before Max_Step, so that 'lose' ends episodes and the step kernel
    restarts UAVs inside the loop.  (Called after the first step, which pops the aliased sub-goal and restarts the segment.)"""
    ms = env.uav_params.max_step
    aged = rng.integers(ms - 50, ms - 1, env.num_UAV).astype(np.int32)
    env.batch.set_state(step=aged)
    if oe is not None:
        oe.ob.step[:] = aged


# (N, capacity): the store wraps on a ragged boundary about every 60 steps
HOST_SIZES = {64: 64 * 60 + 17, 257: 257 * 60 + 100}
HOST_STEPS = 150


@pytest.mark.parametrize("eps", [1.0, 0.3], ids=["eps1", "eps0.3"])
@pytest.mark.parametrize("N", list(HOST_SIZES))
@pytest.mark.parametrize("algo", list(XMLS))
def test_run_step_off_policy_vs_restated_loop(tmp_path, algo, N, eps):
    """Every step of run_step_OffPolicy: the env against the oracle (integers exact, fp64 state 1e-9, reward and observation
    1e-5), the actions against the restated draw of act call t (and the float64 argmax of the parameters before the step on
    greedy rows), the pushed transition group -- s2 of restarted UAVs included -- equal to what the step returned, the gate,
    epoch, Adam step and hard updates against PairedLoop, each update bit for bit against a twin fed the host copy's rows and
    within float64's bounds; arrays returned three steps earlier still hold their values."""
    cap = HOST_SIZES[N]
    env = host_env(tmp_path, algo, N, cap)
    tr, L = env.Trainer, env.Trainer._learner
    assert L.cfg.lockstep_envs == 0 and L.cfg.batch_size == 64
    B, seed = 64, int(L.cfg.seed)
    oe = OracleEnv(env)
    X = twin_of(L)
    M = Mirror(cap, 100)
    loop = R.PairedLoop(M.P, seed, B, update_loop=tr.Update_loop)
    tally = Tally()
    state = env.states()
    assert_obs(state, oe.ob.state(want64=True)[1], "obs0")
    held = collections.deque()
    n_up = n_hard = 0
    for t in range(HOST_STEPS):
        s_in = state.copy()
        before = [L.get_params(w) for w in range(4)]
        ctr = L.counters()
        s2, r, d, info, res = env.run_step_OffPolicy(eps, state)
        what = (algo, N, eps, t)
        # the transition group the step pushed: (s, a, r, s2, d) as the step saw and returned them
        M.P.push(N)
        gs, ga, gr, gs2, gd = L.gather(M.P.newest(N))
        same_rows((gs, gr, gs2, gd), (s_in, r, s2, d.view(np.uint8)), what)
        slots = M.P.slot(M.P.newest(N))
        M.s[slots], M.a[slots], M.r[slots], M.s2[slots], M.d[slots] = gs, ga, gr, gs2, gd
        check_actions(s_in, ga, seed, t, before[0][None], eps, shape_of(L))
        oe.check(env, s2, r, d, info, oe.step(ga), what)
        if t == 0:
            age_episodes(env, np.random.default_rng(N), oe)
        # the learner: PairedLoop's gate and counters, the twin bit for bit, float64
        u = loop.update()
        assert L.counters() == (loop.epoch, loop.adam_t) and res["sum_epoch"] == loop.epoch, (what, L.counters())
        xl = follow(X, u, None if u is None else M.rows(u[1]))
        assert_twins(L, X, res["loss"], xl, what)
        if u is None:
            for w in range(4):
                assert np.array_equal(L.get_params(w), before[w]), (what, w)
        else:
            judge_update(L, before, ctr, M.rows(u[1]), u[0], u[2], float(res["loss"]), tally)
            n_up += 1; n_hard += u[2]
        # _host_out: a returned array stays valid for the next 3 calls (one Move_Agents call per step when state is passed)
        held.append([(x, x.copy()) for x in (s2, r, d, info)])
        if len(held) > 3:
            for x, c in held.popleft():
                assert np.array_equal(x, c), (what, "array of step t - 3 overwritten")
        state = s2
    tally.check()
    assert oe.restarts > 0 and n_up == loop.adam_t == HOST_STEPS - (N <= B) and n_hard >= 49
    assert M.P.count == cap and HOST_STEPS * N >= 2 * cap + N                    # wrapped at least twice
    env.batch.close(); L.close(); X.close()


def test_run_step_state_none_equals_state_passed(tmp_path):
    """run_step_OffPolicy(eps) re-observes the env; passing the previous s2 back must give the same run bit for bit (the
    observation the step returned is the env's state, restarted UAVs included)."""
    N, cap, T = 64, 64 * 20 + 5, 60
    a = host_env(tmp_path, "ddqn", N, cap)
    b = host_env(tmp_path, "ddqn", N, cap)
    state = a.states()
    for t in range(T):
        s2a, ra, da, ia, resa = a.run_step_OffPolicy(0.3, state)
        s2b, rb, db, ib, resb = b.run_step_OffPolicy(0.3)
        same_rows((s2a, ra, da, ia), (s2b, rb, db, ib), t)
        assert float(resa["loss"]) == float(resb["loss"]) and resa["sum_epoch"] == resb["sum_epoch"] == t + 1
        state = s2a
        if t == 0:
            for e in (a, b):
                age_episodes(e, np.random.default_rng(1))
            state = a.states()
    for w in range(4):
        assert np.array_equal(a.Trainer._learner.get_params(w), b.Trainer._learner.get_params(w)), w
    same_rows(a.Trainer._learner.gather(np.arange(cap)), b.Trainer._learner.gather(np.arange(cap)), "store")
    assert (a.batch.get_state()["scenario"] != np.arange(N)).sum() >= N // 2        # restarted inside the step kernel
    for e in (a, b):
        e.batch.close(); e.Trainer._learner.close()


# ------------------------------------------------------------------ (e) the e2e workload as the benchmark builds it
def test_e2e_workload_matches_hand_composed_loop(tmp_path):
    """4 096 UAVs, Batch_Size 4 096, replay 64 x 4 096, QValue3 under DQN, host_driven = 1, seed 42: 5 warm-up steps and 70
    more (the store wraps once) through run_step_OffPolicy, every step bit-identical to observe / act / step / push / update
    on engine objects; the updates of steps 6, 40 and 70 within float64's bounds."""
    N = B = 4096
    cap = 64 * N
    with env_plugin(tmp_path, Batch_Size=str(B), replay_size=str(cap), NetWork="QValueNet_SAC", save_loop="1000000000") as mod:
        env = mod.PathPlan_City_B200(env_dict(XMLS["dqn"], num_UAV=str(N), num_trainers="1", scenario_pool="2048", device="0",
                                              host_driven="1", seed="42"))
    tr, L = env.Trainer, env.Trainer._learner
    assert type(tr).__name__ == "DQN_Trainer_B200" and L.hidden == [64, 64] and L.cfg.algo == engine.ALGO_DQN
    # the same loop on engine objects
    tenv = engine.EnvBatch(env.city, env.uav_params, N, max_subgoals=64, auto_reset=True)
    sc = tenv.make_scenarios(env.pool_size, seed=42, rrt_step=env.sub_granularity)
    tenv.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    tenv.reset(0)
    TL = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DQN, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3,
                        replay_capacity=cap, seed=42)
    TL.init_params(42)
    for w in range(4):
        assert np.array_equal(L.get_params(w), TL.get_params(w)), w
    tloss = torch.zeros(1, device="cuda")
    P = R.Paired(cap)
    loop = R.PairedLoop(P, 42, B, update_loop=3)
    tally = Tally()
    eps = 0.1
    state = env.states()
    tobs = tenv.observe()
    assert np.array_equal(state, tobs.cpu().numpy())
    for step in range(1, 76):
        before = [L.get_params(w) for w in range(4)]
        ctr = L.counters()
        state, r, d, info, res = env.run_step_OffPolicy(eps, state)
        ta = TL.act(tobs, eps, is_train=True)
        out = tenv.step(ta)
        TL.push(tobs, ta, out["reward"], out["obs"], out["done"])
        TL.update(loss=tloss)
        tobs = out["obs"]
        P.push(N)
        u = loop.update()
        torch.cuda.synchronize()
        same_rows((state, r, d.view(np.uint8), info), tuple(out[k].cpu().numpy() for k in ("obs", "reward", "done", "info")), step)
        assert np.array_equal(L.gather(P.newest(N))[1], ta.cpu().numpy()), step
        assert L.counters() == TL.counters() == (loop.epoch, loop.adam_t), step
        for w in range(4):
            assert np.array_equal(L.get_params(w), TL.get_params(w)), (step, w)
        if u is not None:
            assert np.float32(float(res["loss"])) == np.float32(float(tloss)), step
        if step in (6, 40, 70):
            assert u is not None
            judge_update(L, before, ctr, L.gather(u[1]), u[0], u[2], float(res["loss"]), tally)
    tally.check()
    assert P.count == cap and 75 * N > cap
    env.batch.close(); L.close(); tenv.close(); TL.close()


# ------------------------------------------------------------------ (f) prioritised replay through the facade after the wrap
def test_prioritised_facade_after_wrap(dqn_golden, tmp_path):
    """Push_Replay(exp, error) of 2.5 x replay_size transitions in ragged chunks; after each, replay_memory.sample2 returns the
    rows stored at the slots it reports (bit for bit), tree indices slot + capacity - 1, and the oracle SumTree's indices and
    weights on the restated uniforms of that call; update(transition_dict) with idx / weights then rewrites exactly the
    sampled leaves, to min(|Q - y| + 0.01, 1)^0.6 of the float64 update."""
    cap, B = 1000, 64
    tr = trainer_plugin(tmp_path, "Trainer_DDQN_B200.xml", IsPriority_Replay="1", replay_size=str(cap), Batch_Size=str(B))
    L = tr._learner
    seed = int(L.cfg.seed)
    layers = net_layers(100, [64, 64], 27, False)
    M = Mirror(cap, 100)
    rng = np.random.default_rng(17)
    prio = np.zeros(cap, np.float32)
    chunks, total = [250], 250                # a first chunk whose priorities total more than 1 (SumTree.total() is int(tree[0]))
    while total < int(2.5 * cap):
        n = int(rng.choice([1, 37, 250, 333, cap]))
        chunks.append(n); total += n
    n_wrapped = n_partial = 0
    for call, n in enumerate(chunks):
        s, a, r, s2, d = obs_rows(dqn_golden, rng, n, 27)
        err = rng.gamma(1.5, 0.4, n).astype(np.float32)
        tr.Push_Replay((s, a, r.reshape(-1, 1), s2, d.astype(bool).reshape(-1, 1)), torch.tensor(err))
        slots = M.push(s, a, r, s2, d)
        assert tr._head == M.P.head
        prio[slots] = (np.abs(err) + np.float32(0.01)) ** np.float32(0.6)
        leaves, _, _ = L.per_state(cap)
        np.testing.assert_allclose(leaves, prio, rtol=3e-6)
        n_wrapped += M.P.count == cap and M.P.head != 0
        n_partial += M.P.count < cap
        # sample2: slots from the device tree on this call's uniforms
        bs, ba, br, bs2, bd, idx, w = tr.replay_memory.sample2(B)
        idx = np.asarray(idx, np.int64)
        got_slots = idx - (cap - 1)
        same_rows((bs, np.asarray(ba, np.int32), np.asarray(br, np.float32), bs2, np.asarray(bd, np.uint8)),
                  (M.s[got_slots], M.a[got_slots], M.r[got_slots], M.s2[got_slots], M.d[got_slots]), ("sample2", call))
        per = O.OraclePer(cap)
        per.add(leaves[:M.P.count])
        for _ in range(call):                                   # beta advances once per sampling call
            per.sample(np.zeros(1))
        idx_o, w_o, beta_o = per.sample(R.per_uniforms(seed, call, B))
        assert np.array_equal(idx, idx_o), ("tree indices", call)
        np.testing.assert_allclose(w, w_o, rtol=2e-6, err_msg="weights %d" % call)
        before = L.per_state(cap)[0]
        assert L.per_state(cap)[2] == beta_o
        # update(transition_dict) refreshes exactly the sampled leaves
        local, target = L.get_params(0), L.get_params(1)
        tr.update({"states": bs, "actions": ba, "next_states": bs2, "rewards": br, "dones": bd, "idx": idx.tolist(), "weights": w})
        after = L.per_state(cap)[0]
        touched = np.zeros(cap, bool); touched[got_slots] = True
        assert np.array_equal(after[~touched], before[~touched]), call
        _, _, ae, y = f64_update(layers, engine.ALGO_DDQN, False, local, target, bs, np.asarray(ba), np.asarray(br, np.float32), bs2,
                                 np.asarray(bd, np.float32), w=w, gamma=GAMMA)
        # leaves written once, off double-DQN next-state ties (|Q - y| jumps there)
        ql = np.sort(f64_forward(f64_unpack(layers, local), False, bs2)[0], 1)
        clear = ((ql[:, -1] - ql[:, -2]) >= 1e-4) | (np.asarray(bd) != 0)
        once = np.flatnonzero((np.bincount(got_slots, minlength=cap)[got_slots] == 1) & clear)
        assert once.size >= B // 2, call
        x = np.minimum(ae[once] + 0.01, 1.0)                   # ReplayTree.batch_update: min(|e| + eps, upper) ** alpha
        want = x ** 0.6
        tol = 0.6 * x ** -0.4 * abs_err_bound(y[once], np.asarray(br)[once], ae[once]) * 1.01 + 3e-6 * want
        got = after[got_slots[once]]
        assert (np.abs(got - want) <= tol).all(), (call, float(np.abs(got - want).max()))
        prio = after.astype(np.float32)
    assert n_wrapped >= 2 and n_partial >= 1 and sum(chunks) >= 2.5 * cap
    L.close()


# ------------------------------------------------------------------ the refusal
def test_host_driven_refuses_the_sac_trainer(tmp_path):
    """host_driven = 1 with SAC_Trainer_B200 is refused at construction: the host-driven step needs the DQN family's replay
    facade and learn_off_policy."""
    with env_plugin(tmp_path) as mod:
        with pytest.raises(ValueError, match="DQN-family"):
            mod.PathPlan_City_B200(env_dict("Trainer_SAC_B200.xml", "UAV_continuous_B200.xml", num_UAV="8", num_trainers="1",
                                            host_driven="1"))
