"""The updates the lockstep loops sample for themselves (uavrl_train_run, uavrl_sac_train_run): the batch indices, the eps-greedy
actions and SAC's noise restated on the host (tests/replay_restatement.py), and every in-loop update compared with float64.

Every other comparison of these loops runs the same sampler on both sides; here the sampling key and counter, the ring's
oldest frame and per-trainer count, the skip rule, the trainer offsets and the dependent-launch ordering of the loop are
each pinned against an independent statement of them.

A sampled row cannot be redrawn, so two cases are handled where they occur: a row with a hidden pre-activation of the
float64 network within fp32 noise of the ReLU kink exempts only the gradient entries it can move (that unit's weights and
bias and the layers below it), and a double-DQN next state whose two best local values tie within 1e-4 widens the bounds by
what choosing the other action would change, computed from that row's own float64 gradient.  Both are counted and must stay
rare; no tolerance is loosened for the whole batch."""
import numpy as np
import pytest
import torch

import oracle as O
import replay_restatement as R
from gpu_util import city_and_params, dev, n_sm  # noqa: F401  (module fixture)
from qnet_restatement import Tally, check_actions, f64_forward, f64_unpack, f64_update, net_layers, tie_allowance, trunk_exempt
from sac_restatement import HP, check_step, near_decision, read_state, sac_update64
from shapes import SHAPES, SHIPPED, expected_route
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

LR, GAMMA = 5e-4, 0.99


@pytest.fixture(scope="module")
def world(env_golden, env27_golden):
    return city_and_params(env_golden, env27_golden)[:2]


def make_env(world, N, seed=8):
    city, params = world
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(1024, seed=seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    return env


def copy_learner(L, B, algo, shape, tc, G):
    """A learner without a ring in L's state (parameters, target, Adam moments, counters): the twin an explicit batch updates."""
    in_dim, hidden, n_actions, dueling = shape
    X = engine.Learner(in_dim, hidden, n_actions, dueling, algo, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3,
                       replay_capacity=max(1000, 2 * B * G), seed=L.cfg.seed, trainers=G)
    X.set_tensor_cores(tc)
    for w in range(4):
        X.set_params(L.get_params(w), w)
    X.set_counters(*L.counters())
    return X


def gather_batch(L, ring, idx):
    """Rows of trainer-local indices idx[g] for every trainer, stacked in trainer order (update_batch's G blocks)."""
    J = np.concatenate([ring.logical(idx[g], g) for g in range(len(idx))])
    return L.gather(J)


def explicit_update(X, batch, G):
    s, a, r, s2, d = batch
    loss = torch.zeros(G, device="cuda")
    X.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), loss)
    return loss


# ------------------------------------------------------------------ (a) the sampled indices, bit for bit
@pytest.mark.parametrize("G", [1, 3])
def test_qnet_ring_update_samples_restated_indices(world, G):
    """update() without a tape (the loop's Philox draw) equals update_batch on the rows of the restated indices, bit for bit:
    parameters, target, Adam moments, loss and counters; with the ring not yet full, just wrapped and wrapped several times."""
    N, B, cap_frames, seed = 96, 64, 4, 3
    shape = (100, [64, 64], 27, False)
    env = make_env(world, N)
    L = engine.Learner(*shape, engine.ALGO_DDQN, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3, replay_capacity=N * cap_frames,
                       lockstep_envs=N, seed=seed, trainers=G)
    L.init_params(2)
    ring = R.Ring(N * cap_frames, N, G)
    assert ring.ring_frames == cap_frames + 1
    done = 0
    for total in (3, 5, 17):                      # 3 of 4 frames; wrapped once (oldest = 1); wrapped four times
        engine.train_run(env, L, total - done, eps=0.5, do_update=False)
        for _ in range(total - done):
            ring.commit()
        done = total
        assert L.replay_size() == ring.count and ring.count_g() > B
        for _ in range(2):                        # two epochs per state: the counter moves the draw
            X = copy_learner(L, B, engine.ALGO_DDQN, shape, True, G)
            epoch = L.counters()[0] + 1
            idx = [R.sample(seed, epoch, ring.count_g(), B, g) for g in range(G)]
            loss = torch.zeros(G, device="cuda")
            L.update(loss=loss)
            xl = explicit_update(X, gather_batch(L, ring, idx), G)
            torch.cuda.synchronize()
            assert np.array_equal(loss.cpu().numpy(), xl.cpu().numpy()), (total, epoch)
            for w in range(4):
                assert np.array_equal(L.get_params(w), X.get_params(w)), (total, epoch, w)
            assert L.counters() == X.counters() == (epoch, L.counters()[1])
            X.close()
    env.close(); L.close()


@pytest.mark.parametrize("G", [1, 3])
def test_sac_ring_update_samples_restated_indices(world, G):
    """update_replay() without a tape equals update_batch on the rows of the restated indices, bit for bit (the Philox noise is
    keyed alike on both sides); three ring states as for the Q-network learner."""
    N, B, cap_frames, seed = 96, 64, 4, 9
    env = make_env(world, N)
    S = engine.SacLearner(batch_size=B, replay_capacity=N * cap_frames, lockstep_envs=N, seed=seed, trainers=G, **HP)
    S.init_params(4)
    ring = R.Ring(N * cap_frames, N, G)
    done = 0
    for total in (3, 5, 17):
        engine.sac_train_run(env, S, total - done, do_update=False)
        for _ in range(total - done):
            ring.commit()
        done = total
        assert S.replay_size() == ring.count
        X = engine.SacLearner(batch_size=B, seed=seed, trainers=G, **HP)
        for role in range(11):
            X.set_params(role, S.get_params(role))
        sc = S.scalars()
        X.set_scalars(sc["log_alpha"], sc["la_m"], sc["la_v"], sc["epoch"], sc["adam_step"])
        X.set_alpha(S.alpha())
        idx = [R.sample(seed, sc["epoch"] + 1, ring.count_g(), B, g) for g in range(G)]
        s, a, r, s2, d = S.gather(np.concatenate([ring.logical(idx[g], g) for g in range(G)]))
        l_ring, l_batch = torch.zeros(4 * G, device="cuda"), torch.zeros(4 * G, device="cuda")
        S.update_replay(losses=l_ring)
        X.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), losses=l_batch)
        torch.cuda.synchronize()
        assert np.array_equal(l_ring.cpu().numpy(), l_batch.cpu().numpy()), total
        for role in range(14):
            assert np.array_equal(S.get_params(role), X.get_params(role)), (total, role)
        assert S.scalars() == X.scalars() and np.array_equal(S.alpha(), X.alpha())
        X.close()
    env.close(); S.close()


# ------------------------------------------------------------------ (b) the Q-network loop, update by update, against float64
def run_qnet_loop(world, shape, algo, tc, B, N, U, n_iters, cap_frames, G=1, eps=0.3, seed=3, route=None, n_sm=None, fused=None):
    """n_iters calls of train_run(1 iteration, updates_per_iter = U), each checked against the restated schedule, the float64
    update and the oracle's chain from the learner's state before the iteration."""
    in_dim, hidden, n_actions, dueling = shape
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    n_trunk = len(hidden)
    env = make_env(world, N)
    L = engine.Learner(in_dim, hidden, n_actions, dueling, algo, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3,
                       replay_capacity=N * cap_frames, lockstep_envs=N, seed=seed, trainers=G)
    L.init_params(1)
    if route is not None:
        assert L.set_tensor_cores(tc) == (tc and route[0] is not None)
        assert L.route(B) == expected_route(route, B, n_sm, tc)
    else:
        assert L.set_tensor_cores(tc) == tc
        r = L.route(B)
        assert r["td_fused"] == (tc and bool(fused)) and r["train_rows"] == (None if not tc else 64 if B > 32 * n_sm else 32)
    ring = R.Ring(N * cap_frames, N, G)
    loop = R.Loop(ring, seed, B, update_loop=3)
    net = O.make_net(in_dim, hidden, n_actions, int(dueling))
    tally = Tally()
    skipped = hard_seen = wrapped = 0
    loss_t = torch.zeros(G, device="cuda")
    for it in range(n_iters):
        before = [L.get_params(w).reshape(G, -1) for w in range(4)]
        ctr = L.counters()
        st = engine.train_run(env, L, 1, eps, updates_per_iter=U)
        ups = loop.iteration(U)
        wrapped |= ring.head == 0
        assert L.counters() == (loop.epoch, ctr[1] + sum(u is not None for u in ups)), (it, L.counters())
        assert st.updates == sum(u is not None for u in ups)
        s_new, a_new, _, _, _ = L.gather(ring.newest())
        check_actions(s_new, a_new, L.cfg.seed, loop.act_calls - 1, before[0], eps, shape, G)
        after = [L.get_params(w).reshape(G, -1) for w in range(4)]
        if all(u is None for u in ups):
            skipped += 1
            for w in range(4):
                assert np.array_equal(after[w], before[w]), (it, w)
            continue
        losses64, lal_last = np.zeros(G), np.zeros(G)
        for g in range(G):
            OL = O.OracleLearner(net, algo, before[0][g], gamma=GAMMA, lr=LR, update_loop=3)
            OL.target[:] = before[1][g]; OL.m[:] = before[2][g]; OL.v[:] = before[3][g]; OL.t.value = ctr[1]
            allow = np.zeros(L.P)
            first = True
            for u in ups:
                if u is None:
                    continue
                epoch, idx, hard = u
                hard_seen += hard
                batch = L.gather(ring.logical(idx[g], g))
                s, a, r, s2, d = batch
                d = d.astype(np.float32)
                P64 = f64_unpack(layers, OL.local)
                l64, g64 = f64_update(layers, algo, dueling, OL.local, OL.target, s, a, r, s2, d, gamma=GAMMA)[:2]
                kmask, krows = trunk_exempt(layers, n_trunk, P64, dueling, s)
                lal, gal, trows = tie_allowance(layers, algo, dueling, OL.local, OL.target, (s, a, r, s2, d), L.P)
                tally.rows += B; tally.kink_rows += krows; tally.tie_rows += trows
                tally.entries += L.P; tally.exempt += int((kmask | (gal > 0)).sum())
                if U == 1 and first:
                    gg = L.get_params(4).reshape(G, -1)[g].astype(np.float64)
                    err = np.abs(gg - g64) - (2e-4 * np.abs(g64) + 2e-5 + gal)
                    err[kmask] = 0
                    assert (err <= 0).all(), (it, g, float(err.max()), int(err.argmax()))
                OL.epoch = epoch - 1
                lo, _ = OL.update(s, a, r, s2, d)
                assert abs(lo - l64) <= 2e-5 * abs(l64) + lal, (it, g, lo, l64)
                losses64[g], lal_last[g] = l64, lal
                allow = np.maximum(allow, np.where(kmask | (gal > 0) | ((np.abs(g64) < 1e-5) & (g64 != 0)), 4 * LR, 0.0))
                first = False
            for got, want in ((after[0][g], OL.local), (after[1][g], OL.target)):
                dp = np.abs(got - want)
                assert (dp <= np.maximum(2e-5, allow)).all(), (it, g, float(dp.max()), int(dp.argmax()))
            if ups[-1] is not None and ups[-1][2]:
                assert np.array_equal(after[1][g], after[0][g])          # hard update landed on this epoch
            elif all(u is None or not u[2] for u in ups):
                assert np.array_equal(after[1][g], before[1][g])
        if ups[-1] is not None:
            lt = float(st.last_loss)
            # the loop reports the mean over trainers of each trainer's last loss; with U = 3 the float64 loss is taken from the
            # oracle's chain before the last update
            assert abs(lt - losses64.mean()) <= 2e-5 * abs(losses64.mean()) + lal_last.mean(), (it, lt, losses64)
    tally.check()
    env.close(); L.close()
    return dict(skipped=skipped, hard=hard_seen, wrapped=wrapped)


NETS = {"dqn": (SHIPPED[0], engine.ALGO_DQN), "ddqn": (SHIPPED[0], engine.ALGO_DDQN), "dueling": (SHIPPED[2], engine.ALGO_DUELING)}

# (net, tensor cores, B, N, updates per iteration, fused TD): 32-row training tiles (B = 64) with the TD pass fused, 64-row
# tiles (B = 4 500 > 32 x 132) fused, and separate TD passes
LOOP_LEGS = {
    "dqn-B64": ("dqn", True, 64, 48, 1, 1),
    "ddqn-B64": ("ddqn", True, 64, 48, 1, 1),
    "dueling-B64": ("dueling", True, 64, 48, 1, 1),
    "ddqn-B64-fp32": ("ddqn", False, 64, 48, 1, 1),
    "ddqn-B64-U3": ("ddqn", True, 64, 48, 3, 1),
    "dueling-B64-U3-fp32": ("dueling", False, 64, 48, 3, 1),
    "ddqn-B64-sepTD": ("ddqn", True, 64, 48, 1, 0),
    "ddqn-B4500": ("ddqn", True, 4500, 2048, 1, 1),
    "dqn-B4500-sepTD": ("dqn", True, 4500, 2048, 1, 0),
}


@pytest.mark.parametrize("leg", list(LOOP_LEGS))
def test_qnet_loop_updates_vs_float64(world, leg, n_sm):
    """The shipped networks in the loop: warm-up iterations (count <= B) advance only the epoch, every update equals float64 /
    the oracle on the restated rows, hard target updates land on every third epoch, and the ring wraps."""
    name, tc, B, N, U, fuse = LOOP_LEGS[leg]
    shape, algo = NETS[name]
    try:
        _lib.lib().uavrl_set_fuse_td(fuse)
        n_iters = 9 if B <= 64 else 7
        out = run_qnet_loop(world, shape, algo, tc, B, N, U, n_iters, cap_frames=4, n_sm=n_sm, fused=fuse)
    finally:
        _lib.lib().uavrl_set_fuse_td(1)
    assert out["skipped"] >= 1 and out["hard"] >= 1 and out["wrapped"]


ROUTE_SHAPES = {                       # one shape of each route of shapes.SHAPES with in_dim 100 (the UAV observation)
    "generic": next(s for s in SHAPES if s[0] == 100 and s[4][:2] == ("generic", "generic")),
    "tc_td_fp32_update": next(s for s in SHAPES if s[0] == 100 and s[4][0] is not None and s[4][1] is None),
    "fp32": next(s for s in SHAPES if s[0] == 100 and s[4][0] is None),
}


@pytest.mark.parametrize("route_name", list(ROUTE_SHAPES))
def test_qnet_loop_routes_vs_float64(world, route_name, n_sm):
    in_dim, hidden, n_actions, dueling, route = ROUTE_SHAPES[route_name]
    out = run_qnet_loop(world, (in_dim, hidden, n_actions, bool(dueling)), engine.ALGO_DDQN, True, 64, 48, 1, 9, cap_frames=4,
                        route=route, n_sm=n_sm)
    assert out["skipped"] >= 1 and out["wrapped"]


# ------------------------------------------------------------------ (d) grouped trainers
def test_grouped_loop_updates_vs_float64(world, n_sm):
    """G = 3 trainers of 40 envs (not a multiple of 32), B = 64: trainers hold 40, 80, ... transitions, so the first iteration
    is skipped per trainer although the ring holds 120 > 64; each trainer's update against float64 on its own restated rows."""
    out = run_qnet_loop(world, (100, [64, 64], 27, False), engine.ALGO_DDQN, True, 64, 120, 1, 8, cap_frames=4, G=3, n_sm=n_sm, fused=1)
    assert out["skipped"] == 1 and out["wrapped"]


# ------------------------------------------------------------------ (c) across iterations, with dependent launches
@pytest.mark.parametrize("pdl,fuse_td", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_loop_call_matches_twin_replay(world, pdl, fuse_td):
    """One train_run call of 20 iterations (act -> env step -> update, programmatic dependent launch on or off, TD fused or
    not) ends in the bits of a twin learner that replays the restated updates through update_batch on the gathered rows; the
    twin's chain stays within the oracle's bounds at every step.  The ring (24 frames) does not wrap, so every transition the
    loop sampled is still readable afterwards."""
    N, B, seed, n_iters, eps = 256, 384, 5, 20, 0.2
    shape, algo = NETS["ddqn"]
    try:
        _lib.lib().uavrl_set_pdl(pdl)
        _lib.lib().uavrl_set_fuse_td(fuse_td)
        env = make_env(world, N)
        L = engine.Learner(*shape, algo, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3, replay_capacity=N * 24, lockstep_envs=N,
                           seed=seed)
        L.init_params(3)
        assert L.td_fused() == bool(fuse_td)
        X = copy_learner(L, B, algo, shape, True, 1)
        engine.train_run(env, L, n_iters, eps=eps)
        torch.cuda.synchronize()
        assert L.replay_size() == n_iters * N
        ring = R.Ring(N * 24, N)
        loop = R.Loop(ring, seed, B, update_loop=3)
        net = O.make_net(100, [64, 64], 27, 0)
        layers = net_layers(100, [64, 64], 27, False)
        n_up = 0
        for k in range(n_iters):
            # iteration k acted with the weights after iteration k - 1's update: the twin holds them now.  The ring grows by N
            # per iteration and never wraps, so iteration k's transitions are whole-ring indices [k N, (k + 1) N)
            (u,) = loop.iteration(1)
            s, a, _, _, _ = L.gather(np.arange(k * N, (k + 1) * N))
            greedy, ra = R.eps_greedy(seed, k, N, eps, 27)
            assert np.array_equal(a[~greedy], ra[~greedy]), k
            q = f64_forward(f64_unpack(layers, X.get_params(0)), False, s)[0]
            top2 = np.sort(q, 1)[:, -2:]
            clear = greedy & ((top2[:, 1] - top2[:, 0]) > 1e-4)
            assert clear.sum() >= 0.97 * greedy.sum() and np.array_equal(a[clear], q[clear].argmax(1)), k
            if u is None:
                X.set_counters(X.counters()[0] + 1, X.counters()[1])
                continue
            epoch, idx, _ = u
            assert ring.count == (k + 1) * N and ring.oldest() == 0
            batch = L.gather(idx[0])
            s, a, r, s2, d = batch
            OL = O.OracleLearner(net, algo, X.get_params(0), gamma=GAMMA, lr=LR, update_loop=3)
            OL.target[:] = X.get_params(1); OL.m[:] = X.get_params(2); OL.v[:] = X.get_params(3); OL.t.value = X.counters()[1]
            OL.epoch = epoch - 1
            l64, g64 = f64_update(layers, algo, False, X.get_params(0), X.get_params(1), s, a, r, s2, d.astype(np.float32), gamma=GAMMA)[:2]
            lal, gal, _ = tie_allowance(layers, algo, False, X.get_params(0), X.get_params(1), (s, a, r, s2, d.astype(np.float32)), X.P)
            kmask, _ = trunk_exempt(layers, 2, f64_unpack(layers, X.get_params(0)), False, s)
            xl = explicit_update(X, batch, 1)
            lo, _ = OL.update(s, a, r, s2, d.astype(np.float32))
            torch.cuda.synchronize()
            assert X.counters()[0] == epoch
            assert abs(float(xl) - l64) <= 2e-5 * abs(l64) + lal, (epoch, float(xl), l64)
            allow = np.where(kmask | (gal > 0) | ((np.abs(g64) < 1e-5) & (g64 != 0)), 4 * LR, 2e-5)
            for got, want in ((X.get_params(0), OL.local), (X.get_params(1), OL.target)):
                assert (np.abs(got - want) <= allow).all(), (epoch, float(np.abs(got - want).max()))
            n_up += 1
        assert n_up == n_iters - 1 and L.counters() == X.counters() == (n_iters, n_iters - 1)
        for w in range(4):
            assert np.array_equal(L.get_params(w), X.get_params(w)), w
        env.close(); L.close(); X.close()
    finally:
        _lib.lib().uavrl_set_pdl(1)                 # library defaults: PDL on, fused TD on
        _lib.lib().uavrl_set_fuse_td(1)


# ------------------------------------------------------------------ (e) the SAC loop
SAC_STATE = ("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v")


@pytest.mark.parametrize("obs,hid", [(100, 64), (100, 32)])
def test_sac_loop_updates_vs_float64(world, obs, hid):
    """sac_train_run one iteration at a time: warm-up iterations advance the epoch only; every update equals the float64 SAC
    step on the restated rows with the restated noise (check_step's bounds), log_alpha and the Adam step included."""
    N, B, seed, cap_frames = 48, 64, 9, 4
    assert obs == 100                                   # the env's observation
    env = make_env(world, N)
    S = engine.SacLearner(hidden=hid, batch_size=B, replay_capacity=N * cap_frames, lockstep_envs=N, seed=seed, **HP)
    S.init_params(5)
    ring = R.Ring(N * cap_frames, N)
    loop = R.Loop(ring, seed, B)
    n_checked = skipped = n_near = n_exempt = n_rows = 0
    for it in range(12):
        prev = read_state(S)
        sc0 = S.scalars()
        st = engine.sac_train_run(env, S, 1)
        (u,) = loop.iteration(1)
        sc = S.scalars()
        assert sc["epoch"] == loop.epoch
        if u is None:
            skipped += 1
            assert dict(sc, epoch=0) == dict(sc0, epoch=0) and st.updates == 0
            got = read_state(S)
            for k in SAC_STATE:
                assert np.array_equal(got[k], prev[k]), (it, k)
            continue
        epoch, idx, _ = u
        s, a, r, s2, d = S.gather(ring.logical(idx[0], 0))
        c_next, c_cur = R.sac_update_ctrs(epoch)
        e1, e2 = R.sac_noise(seed, c_next, B), R.sac_noise(seed, c_cur, B)
        new, out = sac_update64(prev, s, a, r, s2, d.astype(np.float64), e1, e2, obs, hid, 1.0)
        near, near_actor = near_decision(out)
        n_rows += B
        n_near += int((near | near_actor).sum())
        assert abs(st.last_loss - out["l_actor"]) <= 1e-5 * out["lscale_actor"] + 1e-4 * abs(out["l_actor"]), it
        # the loop reports the actor loss only; the critics are judged by their gradients and parameters
        losses = out["losses"].copy()
        losses[0] = st.last_loss
        try:
            check_step(S, prev, new, out, losses, ("sac", it))
            n_checked += 1
        except AssertionError:
            # only a batch with a row at a ReLU kink or a q1 / q2 tie of the float64 step may miss the bounds
            if not (near.any() or near_actor.any()):
                raise
            n_exempt += 1
    # (a SAC row meets some decision point of its ~500 ReLU units and q1 / q2 pairs far more often than a Q-network row, so the
    # rare thing here is a batch that actually misses the bounds)
    assert skipped == 1 and n_checked + n_exempt == 11 and n_exempt <= 2, (n_checked, n_exempt, n_near, n_rows)
    assert ring.count == 4 * N and ring.head == 12 % 5                      # wrapped: 12 commits through 5 frames
    env.close(); S.close()


# ------------------------------------------------------------------ (f) the benchmark's scale
def test_benchmark_scale_updates(world):
    """bench.py configs[3] per GPU: 8 192 envs, batch 8 192, replay 2^20 (128 frames), double DQN: a 20-bit sampling domain,
    64-row training tiles, fused TD.  The ring is filled by collection-only iterations; then 3 in-loop updates, each equal
    bit for bit to update_batch on the restated rows and within 2e-5 of the float64 loss."""
    N = B = 8192
    seed = 1
    shape, algo = NETS["ddqn"]
    env = make_env(world, N)
    L = engine.Learner(*shape, algo, lr=LR, gamma=GAMMA, batch_size=B, update_loop=3, replay_capacity=1 << 20, lockstep_envs=N, seed=seed)
    L.init_params(0)
    assert L.td_fused() and L.route(B)["train_rows"] == 64
    ring = R.Ring(1 << 20, N)
    assert ring.ring_frames == 129
    engine.train_run(env, L, 130, eps=1.0, do_update=False)
    for _ in range(130):
        ring.commit()
    assert ring.count == 128 * N == L.replay_size() and ring.oldest() == 2
    layers = net_layers(100, [64, 64], 27, False)
    loop = R.Loop(ring, seed, B, update_loop=3, epoch=L.counters()[0], act_calls=130)
    for step in range(3):
        X = copy_learner(L, B, algo, shape, True, 1)
        st = engine.train_run(env, L, 1, eps=0.1)
        (u,) = loop.iteration(1)
        epoch, idx, _ = u
        assert L.counters()[0] == epoch
        batch = L.gather(ring.logical(idx[0]))
        l64 = f64_update(layers, algo, False, X.get_params(0), X.get_params(1), *batch[:4], batch[4].astype(np.float32), gamma=GAMMA)[0]
        lal, _, _ = tie_allowance(layers, algo, False, X.get_params(0), X.get_params(1), batch[:4] + (batch[4].astype(np.float32),), X.P)
        xl = explicit_update(X, batch, 1)
        torch.cuda.synchronize()
        assert float(xl) == st.last_loss, step
        assert abs(float(xl) - l64) <= 2e-5 * abs(l64) + lal, (step, float(xl), l64)
        for w in range(4):
            assert np.array_equal(L.get_params(w), X.get_params(w)), (step, w)
        X.close()
    env.close(); L.close()
