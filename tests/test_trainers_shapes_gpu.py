"""Grouped Q-network trainers (uavrl_learner_create_trainers) at every route of the shape sweep, away from the shipped G = 4.
Every grouped kernel takes its trainer from blockIdx.y and offsets weight images, rows, scratch, sampling keys and partials by
it; with G = 1 every offset is 0, so the shape sweeps alone cannot see a wrong one.  Here trainer g must equal, bit for bit, a
stand-alone learner with its parameters and Adam moments, seed + g, replay_capacity / G and Ng = lockstep_envs / G envs:
actions, Q, its loss slot, local, target, both moments, gradient, counters, ring rows, env state and, with prioritised replay,
sampled slots, weights, leaves, totals and beta.  Every trainer holds distinct parameters, moments and rows, so a trainer that
reads another's data fails.  Bit-identity cannot see a bug the grouped and stand-alone paths share, so on every route the
last trainer (the largest offsets) is also held to float64 with the shape sweeps' tolerances.

Per-trainer sizes reach down to one row (a tile of 31 padding rows in every CTA) and one env (Ng = 1, the layout the env
plug-in's one trainer per UAV gives), G up to 65 535 (gridDim.y's limit); the lockstep loop runs with rings that wrap and
episodes that end, and the launch count per iteration and per update is checked to be that of G = 1."""
import numpy as np
import pytest
import torch

import oracle as O
from fl_restatement import check_rounds
from gpu_util import (DEV, assert_same, assert_trainers_equal, assert_trees_equal, dev, learner, n_sm,  # noqa: F401  (fixture)
                      ring_env, short_episode_env, standalone_like)
from qnet_restatement import abs_err_bound, big_inputs, draw_batch, f64_forward, f64_unpack, f64_update, net_layers
from shapes import ROUTES, SHAPES, SHIPPED, act_sizes, expected_route
from shapes import shape_id as route_id
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

# the lockstep loop steps the 27-action UAV env on the 100-d observation: the routes of ROUTES it can drive
LOOP_ROUTES = [s for s in ROUTES if s[0] == 100 and s[2] == 27]
GENERIC = (100, [64, 32], 27, 1)          # generic forward + generic training kernel
FP32_ONLY = (100, [128, 64, 64], 27, 1)   # no tensor-core kernel at all


def test_tables_cover_every_route():
    """ROUTES keeps one shape of every route of the shape sweep; the loop legs keep the FIXED, generic, tensor-core TD into
    the fp32 update (dual- and single-weights) and fp32-only routes."""
    assert {s[4] for s in SHAPES} <= {s[4] for s in ROUTES}
    loop = {s[4] for s in LOOP_ROUTES}
    assert any(r[0] == "fixed" and r[1] == "fixed" for r in loop)
    assert any(r[0] == "generic" and r[1] == "generic" for r in loop)
    assert any(r[0] is not None and r[1] is None and r[4] for r in loop)
    assert any(r[0] is not None and r[1] is None and not r[4] for r in loop)
    assert any(r[0] is None for r in loop)
    assert all(any(s[:4] == want for s in LOOP_ROUTES) for want in (GENERIC, FP32_ONLY, SHIPPED[0]))


@pytest.fixture(autouse=True)
def restore_switches():
    yield
    _lib.lib().uavrl_set_pdl(1)                 # library defaults: PDL on, fused TD on
    _lib.lib().uavrl_set_fuse_td(1)
    O.set_loss_kind("mse")                      # the oracle's loss kind is process-wide state


def algo_of(name, shape):
    if name == "dqn":
        return engine.ALGO_DQN
    return engine.ALGO_DUELING if shape[3] else engine.ALGO_DDQN


def distinct_moments(L, rng):
    """Adam moments of every trainer drawn apart: a trainer reading another's moments shows in its next step."""
    L.set_params(rng.normal(0, 1e-3, (L.G, L.P)).astype(np.float32), 2)
    L.set_params(np.abs(rng.normal(0, 1e-6, (L.G, L.P))).astype(np.float32), 3)


# ---------------------------------------------------------------------------------------------------------------------
# 1. act at every route
@pytest.mark.parametrize("shape", ROUTES, ids=route_id)
def test_act_equals_standalone_and_float64(dqn_golden, shape, n_sm):
    """G = 3 and 7, per-trainer n = 1, 31, 33, 1000 and (G = 3) the 64- and 128-row tile sizes of the shape sweep; tensor
    cores on and off, epsilon-greedy tapes and Philox draws.  Every trainer bit for bit as its stand-alone learner; the last
    trainer's Q within 2e-5 abs + 2e-5 rel of float64, its greedy actions the float64 argmax wherever the top-2 gap exceeds
    1e-4, its random ones the tape's."""
    in_dim, hidden, n_actions, dueling, route = shape
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    rng = np.random.default_rng([in_dim, sum(hidden), n_actions, 1])
    eps = 0.3
    for G in (3, 7):
        Lg = learner(shape, G)
        Lg.init_params(3)
        solo = [standalone_like(Lg, shape, g) for g in range(G)]
        P64 = f64_unpack(layers, Lg.get_params(0)[G - 1])
        for n in [1, 31, 33, 1000] + (act_sizes(route, n_sm)[1:] if G == 3 else []):
            x = big_inputs(dqn_golden, G * n, rng, in_dim)
            u = rng.random(G * n).astype(np.float32)
            ra = rng.integers(0, n_actions, G * n).astype(np.int32)
            obs, u_d, ra_d = dev(x), dev(u), dev(ra)
            last = slice((G - 1) * n, G * n)
            q64 = f64_forward(P64, dueling, x[last])[0]
            top2 = np.sort(q64, 1)[:, -2:]
            clear = (top2[:, 1] - top2[:, 0]) > 1e-4
            for tc in (True, False):
                for L in [Lg] + solo:
                    assert L.set_tensor_cores(tc) == (tc and route[0] is not None)
                assert Lg.route(n) == expected_route(route, n, n_sm, tc), (G, n, tc)
                a, q = Lg.act(obs, eps, u_tape=u_d, rand_tape=ra_d, want_q=True)
                ap = Lg.act(obs, eps)
                a, q, ap = a.cpu().numpy(), q.cpu().numpy(), ap.cpu().numpy()
                for g, S in enumerate(solo):
                    blk = slice(g * n, (g + 1) * n)
                    a1, q1 = S.act(obs[blk].contiguous(), eps, u_tape=u_d[blk].contiguous(), rand_tape=ra_d[blk].contiguous(),
                                   want_q=True)
                    ap1 = S.act(obs[blk].contiguous(), eps)
                    what = (G, n, tc, g)
                    assert_same(q[blk], q1.cpu().numpy(), ("Q",) + what)
                    assert_same(a[blk], a1.cpu().numpy(), ("actions (tapes)",) + what)
                    assert_same(ap[blk], ap1.cpu().numpy(), ("actions (Philox)",) + what)
                err = np.abs(q[last] - q64) - (2e-5 + 2e-5 * np.abs(q64))
                assert (err <= 0).all(), (G, n, tc, float(err.max()), np.unravel_index(err.argmax(), err.shape))
                rand = u[last] <= eps
                assert np.array_equal(a[last][rand], ra[last][rand]), (G, n, tc)
                greedy = ~rand & clear
                assert np.array_equal(a[last][greedy], q64[greedy].argmax(1)), (G, n, tc)
        for L in [Lg] + solo:
            L.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. explicit updates at every route
VARIANTS = {                              # algorithm ("ddqn" is the dueling trainer on a dueling head), loss, tensor cores
    "dqn-mse": ("dqn", "mse", True),
    "ddqn-huber": ("ddqn", "huber", True),
    "ddqn-mse-fp32": ("ddqn", "mse", False),
}
# per-trainer batches on one handle created with batch_size = 1: every scratch buffer grows (1 -> 33 -> 64 -> 6000), is
# reused at a smaller batch and reused again at the grown size; update_loop = 3 puts a hard target update at steps 3 and 6
GROW_SEQ = [1, 1, 33, 64, 6000, 64, 6000]


def check_last_vs_float64(Lg, layers, algo, dueling, local, target, batch, kind, loss, what):
    """The last trainer's loss slot within 2e-5 relative of float64 and every gradient entry within 2e-4 |g64| + 2e-5 +
    2^-20 S64 (S64: the sum of the magnitudes of the products the entry adds up, test_weighted_update_shapes_gpu).
    Below the shape sweeps' smallest batch (64) the loss may also move by what the fp32 error of q_a - y allows: with
    delta = abs_err_bound (the act tests' bound on Q carried through y), 2 |diff| delta + delta^2 per sample (MSE) or
    min(|diff|, 1) delta (Huber).  At B = 1 the loss is one sample's: no average hides that error, and q_a - y cancels."""
    G = Lg.G
    l64, g64, ae64, y64, mag64 = f64_update(layers, algo, dueling, local, target, *batch, None, kind, abs_terms=True)
    delta = abs_err_bound(y64, batch[2], ae64)
    moved = np.mean(2.0 * ae64 * delta + delta ** 2 if kind == "mse" else np.minimum(ae64, 1.0) * delta)
    tol = 2e-5 * abs(l64) + (moved if len(ae64) < 64 else 0.0)
    assert abs(float(loss[G - 1]) - l64) <= tol, what + (float(loss[G - 1]), l64, tol)
    gg = Lg.get_params(4)[G - 1].astype(np.float64)
    err = np.abs(gg - g64) - (2e-4 * np.abs(g64) + 2e-5 + 2.0 ** -20 * mag64)
    assert (err <= 0).all(), what + (float(err.max()), int(err.argmax()), int((err > 0).sum()))


def run_updates(dqn_golden, shape, variant, G, seq, seed):
    in_dim, hidden, n_actions, dueling, route = shape
    name, kind, tc = VARIANTS[variant]
    algo = algo_of(name, shape)
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    rng = np.random.default_rng([seed, in_dim, sum(hidden), n_actions, algo, sorted(VARIANTS).index(variant)])
    kw = dict(algo=algo, batch_size=seq[0], update_loop=3, loss=kind)
    Lg = learner(shape, G, **kw)
    Lg.init_params(5)
    distinct_moments(Lg, rng)
    solo = [standalone_like(Lg, shape, g, **kw) for g in range(G)]
    for L in [Lg] + solo:
        assert L.set_tensor_cores(tc) == (tc and route[0] is not None)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for step, B in enumerate(seq):
        assert Lg.route(B) == expected_route(route, B, n_sm, tc), (step, B)
        local, target = Lg.get_params(0), Lg.get_params(1)
        # every trainer's block is drawn clear of the ReLU kinks, DDQN next-state ties and the Huber branch point of its own
        # networks (draw_batch): the last block is judged against float64, the others only against their stand-alone twins
        blocks = [draw_batch(dqn_golden, rng, layers, dueling, algo, [local[g]], target[g], B, in_dim, n_actions, kind, False)[:5]
                  for g in range(G)]
        s, a, r, s2, d = (np.concatenate(parts) for parts in zip(*blocks))
        s_d, a_d, r_d, s2_d, d_d = dev(s), dev(a), dev(r), dev(s2), dev(d)
        loss = torch.full((G,), float("nan"), device=DEV)
        Lg.update_batch(s_d, a_d, r_d, s2_d, d_d, loss)
        solo_loss = []
        for g, S in enumerate(solo):
            blk = slice(g * B, (g + 1) * B)
            l1 = torch.zeros(1, device=DEV)
            S.update_batch(s_d[blk].contiguous(), a_d[blk].contiguous(), r_d[blk].contiguous(), s2_d[blk].contiguous(),
                           d_d[blk].contiguous(), l1)
            solo_loss.append(l1.cpu().numpy())
        loss = loss.cpu().numpy()
        assert_trainers_equal(Lg, solo, loss, solo_loss)
        O.set_loss_kind(kind)
        check_last_vs_float64(Lg, layers, algo, dueling, local[G - 1], target[G - 1], blocks[G - 1], kind, loss, (step, B))
    assert Lg.counters() == (len(seq), len(seq))
    for L in [Lg] + solo:
        L.close()


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("shape", ROUTES, ids=route_id)
def test_update_grows_scratch_equals_standalone_and_float64(dqn_golden, shape, variant):
    """G = 3, per-trainer batches 1, 1, 33, 64, 6000, 64, 6000 on one handle (GROW_SEQ): bit for bit as the stand-alone
    learners after every step, the last trainer against float64."""
    run_updates(dqn_golden, shape, variant, 3, GROW_SEQ, 0)


@pytest.mark.parametrize("shape", ROUTES, ids=route_id)
def test_update_b12000_two_trainers(dqn_golden, shape):
    """G = 2 at 12 000 per trainer (64-row training tiles, TD targets in separate passes), 4 steps."""
    run_updates(dqn_golden, shape, "dqn-mse", 2, [12000] * 4, 1)


# ---------------------------------------------------------------------------------------------------------------------
# 3 - 5. the lockstep loop
class LoopRun:
    """A grouped learner on N = G Ng auto-resetting envs run through `iters` lockstep iterations.  The scenario pool holds
    pool_n scenarios with pool_n dividing (G - 1) Ng: grouped env g Ng + j restarts at (g Ng + j + k N) mod pool_n, which is
    where the stand-alone env j of trainer g (Ng envs, reset(g Ng)) restarts, (g Ng + j + k Ng) mod pool_n.  The ring holds
    `frames` frames of Ng transitions per trainer."""

    def __init__(self, env_golden, env27_golden, shape, G, Ng, iters, frames, batch, per=False, pool_n=None, seed=11,
                 tc=True, eps=0.3):
        self.shape, self.G, self.Ng, self.N = shape, G, Ng, G * Ng
        self.iters, self.frames, self.per, self.eps, self.seed = iters, frames, per, eps, seed
        self.city, self.params = short_episode_env(env_golden, env27_golden)
        pool_n = pool_n or Ng
        assert ((G - 1) * Ng) % pool_n == 0
        self.pool = engine.EnvBatch(self.city, self.params, pool_n, max_subgoals=64).make_scenarios(pool_n, seed=5)
        self.kw = dict(algo=algo_of("ddqn", shape), batch_size=batch, update_loop=3)
        self.tc = tc
        rng = np.random.default_rng([G, Ng, seed])
        self.env = ring_env(self.city, self.params, self.N, self.pool, 0)
        self.L = learner(shape, G, seed=seed, replay_capacity=G * frames * Ng, lockstep_envs=self.N, **self.kw)
        self.L.init_params(1)
        distinct_moments(self.L, rng)
        self.init = [self.L.get_params(w) for w in range(4)]
        if per:
            self.L.per_enable_trainers()
        self.L.set_tensor_cores(tc)
        self.st = engine.train_run(self.env, self.L, iters, eps=eps)

    def standalone(self, g):
        e1 = ring_env(self.city, self.params, self.Ng, self.pool, g * self.Ng)
        L1 = learner(self.shape, 1, seed=self.seed + g, replay_capacity=self.frames * self.Ng, lockstep_envs=self.Ng, **self.kw)
        for w in range(4):
            L1.set_params(self.init[w][g], w)
        if self.per:
            L1.per_enable()
        L1.set_tensor_cores(self.tc)
        s1 = engine.train_run(e1, L1, self.iters, eps=self.eps)
        return e1, L1, s1

    def ring_rows(self, g, n_g):
        k = np.arange(n_g, dtype=np.int64)
        return self.L.gather((k // self.Ng) * self.N + g * self.Ng + k % self.Ng)

    def n_slots(self):
        return (self.frames + 1) * self.Ng             # trainer-local slots: ring frames x Ng


def compare_pairs(run, trainers):
    """Trainers `trainers` of run.L against their stand-alone pairs: vectors, counters, env blocks, ring rows, trees and the
    sampler, then one more ring-sampled update (every loss slot against its pair's loss)."""
    L, G, Ng, st = run.L, run.G, run.Ng, run.st
    assert st.updates > 0
    pairs = {g: run.standalone(g) for g in trainers}
    for g, (_, _, s1) in pairs.items():
        assert s1.updates == st.updates, g
    vecs = [L.get_params(w) for w in range(5)]
    sg = run.env.get_state()
    n_g = L.replay_size() // G
    leaves = L.per_state(run.n_slots()) if run.per else None
    for g, (e1, L1, _) in pairs.items():
        for w, what in enumerate(("local", "target", "exp_avg", "exp_avg_sq", "grad")):
            assert_same(vecs[w][g], L1.get_params(w), "%s of trainer %d" % (what, g))
        assert L1.counters() == L.counters()
        s1 = e1.get_state()
        for k in sg:
            assert_same(sg[k][g * Ng:(g + 1) * Ng], s1[k], "env state %s, block %d" % (k, g))
        assert L1.replay_size() == n_g
        for x, y, what in zip(run.ring_rows(g, n_g), L1.gather(np.arange(n_g)), ("s", "a", "r", "s2", "d")):
            assert_same(x, y, "ring %s, trainer %d" % (what, g))
        if run.per:
            l1, t1, b1 = L1.per_state(run.n_slots())
            assert_same(leaves[0][g], l1, "leaves of trainer %d" % g)
            assert_same(leaves[1][g:g + 1], np.array([t1]), "total of trainer %d" % g)
            assert leaves[2] == b1
    if len(pairs) == G:
        losses = [np.float32(s1.last_loss) for _, _, s1 in pairs.values()]
        assert np.float32(st.last_loss) == np.float32(sum(float(x) for x in losses) / G)
    # one more ring-sampled update: every trainer's own loss slot against its pair's loss
    loss = torch.full((G,), float("nan"), device=DEV)
    L.update(loss=loss)
    loss = loss.cpu().numpy()
    vecs = [L.get_params(w) for w in range(5)]
    for g, (_, L1, _) in pairs.items():
        l1 = torch.zeros(1, device=DEV)
        L1.update(loss=l1)
        assert_same(loss[g:g + 1], l1.cpu().numpy(), "loss of trainer %d" % g)
        for w in range(5):
            assert_same(vecs[w][g], L1.get_params(w), "vector %d of trainer %d after the ring update" % (w, g))
    if run.per:
        B = run.kw["batch_size"]
        assert_trees_equal_subset(L, pairs, run.n_slots())
        sl, wt = L.per_sample(B)
        sl, wt = sl.cpu().numpy(), wt.cpu().numpy()
        for g, (_, L1, _) in pairs.items():
            s1, w1 = L1.per_sample(B)
            assert_same(sl[g], s1.cpu().numpy(), "sampled slots of trainer %d" % g)
            assert_same(wt[g], w1.cpu().numpy(), "weights of trainer %d" % g)
    for e1, L1, _ in pairs.values():
        e1.close(); L1.close()
    return n_g


def assert_trees_equal_subset(L, pairs, n_slots):
    if len(pairs) == L.G:
        assert_trees_equal(L, [L1 for _, L1, _ in pairs.values()], n_slots)
        return
    leaves, totals, beta = L.per_state(n_slots)
    for g, (_, L1, _) in pairs.items():
        l1, t1, b1 = L1.per_state(n_slots)
        assert_same(leaves[g], l1, "leaves of trainer %d" % g)
        assert_same(totals[g:g + 1], np.array([t1]), "total of trainer %d" % g)
        assert beta == b1


LOOP_GN = [(4, 37), (16, 3), (64, 1)]
LOOP_ITERS, LOOP_FRAMES, LOOP_BATCH = 40, 24, 16        # the ring wraps; Ng = 1 trainers update from iteration 17 on


@pytest.mark.parametrize("G,Ng", LOOP_GN, ids=["G%d-Ng%d" % gn for gn in LOOP_GN])
@pytest.mark.parametrize("shape", LOOP_ROUTES, ids=route_id)
def test_lockstep_loop_equals_standalone_pairs(env_golden, env27_golden, shape, G, Ng):
    """40 iterations through a 24-frame ring with episodes ending (auto_reset, a pool of exactly Ng scenarios): every trainer
    against its stand-alone pair.  At (16, 3) the loop runs again with dependent launches and the fused TD pass off and must
    end in the same bits."""
    run = LoopRun(env_golden, env27_golden, shape, G, Ng, LOOP_ITERS, LOOP_FRAMES, LOOP_BATCH)
    assert run.st.episodes_ended > 0 and run.st.env_steps == LOOP_ITERS * G * Ng
    assert run.L.replay_size() == G * LOOP_FRAMES * Ng                    # full: the ring wrapped
    if (G, Ng) == (16, 3):
        ref = [run.L.get_params(w) for w in range(5)]
        ring = [run.ring_rows(g, LOOP_FRAMES * Ng) for g in range(G)]
        es = run.env.get_state()
        _lib.lib().uavrl_set_pdl(0)
        _lib.lib().uavrl_set_fuse_td(0)
        off = LoopRun(env_golden, env27_golden, shape, G, Ng, LOOP_ITERS, LOOP_FRAMES, LOOP_BATCH)
        _lib.lib().uavrl_set_pdl(1)
        _lib.lib().uavrl_set_fuse_td(1)
        for w in range(5):
            assert_same(off.L.get_params(w), ref[w], "vector %d with PDL and fused TD off" % w)
        for g in range(G):
            for x, y in zip(off.ring_rows(g, LOOP_FRAMES * Ng), ring[g]):
                assert_same(x, y, "ring of trainer %d with PDL and fused TD off" % g)
        es_off = off.env.get_state()
        for k in es:
            assert_same(es_off[k], es[k], "env state %s with PDL and fused TD off" % k)
        assert off.st.last_loss == run.st.last_loss and off.L.counters() == run.L.counters()
        off.env.close(); off.L.close()
    compare_pairs(run, range(G))
    run.env.close(); run.L.close()


PER_LEGS = [(s, G, Ng) for s in (GENERIC, FP32_ONLY) for G, Ng in ((64, 1), (4, 37))]


@pytest.mark.parametrize("shape,G,Ng", PER_LEGS, ids=["%s-G%d-Ng%d" % ("generic" if s == GENERIC else "fp32", G, Ng)
                                                      for s, G, Ng in PER_LEGS])
def test_lockstep_loop_with_per_equals_standalone_pairs(env_golden, env27_golden, shape, G, Ng):
    """The loop legs with one SumTree per trainer: trees, sampled slots and weights as the stand-alone learners'."""
    full = next(s for s in LOOP_ROUTES if s[:4] == shape)
    run = LoopRun(env_golden, env27_golden, full, G, Ng, LOOP_ITERS, LOOP_FRAMES, LOOP_BATCH, per=True)
    assert run.st.episodes_ended > 0
    compare_pairs(run, range(G))
    run.env.close(); run.L.close()


@pytest.mark.parametrize("per", [False, True], ids=["uniform", "per"])
@pytest.mark.parametrize("shape", [SHIPPED[0], GENERIC], ids=["100-64x64-27", "generic"])
def test_reference_scale_g4096_one_env_per_trainer(env_golden, env27_golden, shape, per):
    """README's benchmark layout: 4096 trainers of one env each, batch 64, run until every trainer holds more than 64
    transitions and updates have run (72 iterations, 80 ring frames).  Trainers 0, 1, 2047, 4094, 4095 and three drawn at
    random against stand-alone pairs, then one more ring-sampled update.  The pool holds 4095 scenarios (it divides
    (G - 1) Ng), so the trainers start from different scenarios."""
    G = 4096
    full = next(s for s in LOOP_ROUTES if s[:4] == shape)
    run = LoopRun(env_golden, env27_golden, full, G, 1, 72, 80, 64, per=per, pool_n=G - 1)
    assert run.st.updates == 72 - 64
    pick = sorted({0, 1, 2047, 4094, 4095} | set(np.random.default_rng(2).choice(G, 3, replace=False).tolist()))
    n_g = compare_pairs(run, pick)
    assert n_g == 72
    run.env.close(); run.L.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. gridDim.y = 65535
def test_largest_trainer_count(dqn_golden):
    """65 535 trainers (the largest n_trainers create_trainers accepts) of a small network: act over one row per trainer and
    one update_batch of one transition per trainer.  The first, middle and last trainers against stand-alone learners.  The
    device is shared, so the footprint is measured on 1024 trainers first and the test is skipped when the free memory
    cannot hold 1.5 times the scaled-up figure."""
    G, shape = 65535, (12, [32], 7, 0)
    in_dim, _, n_actions, _ = shape
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    probe = learner(shape, 1024, batch_size=1, replay_capacity=1024)
    probe.init_params(0)
    x = dev(np.zeros((1024, in_dim), np.float32))
    one = torch.zeros(1024, device=DEV)
    probe.act(x, 0.0)
    probe.update_batch(x, one.int(), one, x, one)
    torch.cuda.synchronize()
    per_1024 = free0 - torch.cuda.mem_get_info()[0]
    probe.close(); del x, one
    torch.cuda.synchronize()
    need = 1.5 * per_1024 * (G / 1024.0) + (256 << 20)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("65 535 trainers need about %.1f GB of device memory; %.1f GB are free" % (need / 1e9, free / 1e9))
    rng = np.random.default_rng(65535)
    Lg = learner(shape, G, batch_size=1, replay_capacity=G, algo=engine.ALGO_DDQN)
    vec = [rng.normal(0, 0.3, (G, Lg.P)).astype(np.float32) for _ in range(2)]
    vec += [rng.normal(0, 1e-3, (G, Lg.P)).astype(np.float32), np.abs(rng.normal(0, 1e-6, (G, Lg.P))).astype(np.float32)]
    for w in range(4):
        Lg.set_params(vec[w], w)
    pick = (0, G // 2, G - 1)
    solo = {}
    for g in pick:
        S = learner(shape, 1, 7 + g, batch_size=1, replay_capacity=1, algo=engine.ALGO_DDQN)
        for w in range(4):
            S.set_params(vec[w][g], w)
        solo[g] = S
    x = rng.normal(0, 1, (G, in_dim)).astype(np.float32)
    u = rng.random(G).astype(np.float32)
    ra = rng.integers(0, n_actions, G).astype(np.int32)
    obs = dev(x)
    a, q = Lg.act(obs, 0.3, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
    ap = Lg.act(obs, 0.3)
    a, q, ap = a.cpu().numpy(), q.cpu().numpy(), ap.cpu().numpy()
    for g, S in solo.items():
        a1, q1 = S.act(obs[g:g + 1].contiguous(), 0.3, u_tape=dev(u[g:g + 1]), rand_tape=dev(ra[g:g + 1]), want_q=True)
        assert_same(q[g:g + 1], q1.cpu().numpy(), "Q of trainer %d" % g)
        assert_same(a[g:g + 1], a1.cpu().numpy(), "actions (tapes) of trainer %d" % g)
        assert_same(ap[g:g + 1], S.act(obs[g:g + 1].contiguous(), 0.3).cpu().numpy(), "actions (Philox) of trainer %d" % g)
    s2 = dev(rng.normal(0, 1, (G, in_dim)).astype(np.float32))
    act = dev(rng.integers(0, n_actions, G).astype(np.int32))
    r = dev(rng.normal(0, 1, G).astype(np.float32))
    d = dev((rng.random(G) < 0.2).astype(np.float32))
    loss = torch.full((G,), float("nan"), device=DEV)
    Lg.update_batch(obs, act, r, s2, d, loss)
    loss = loss.cpu().numpy()
    assert np.isfinite(loss).all()
    vecs = [Lg.get_params(w) for w in range(5)]
    for g, S in solo.items():
        l1 = torch.zeros(1, device=DEV)
        S.update_batch(obs[g:g + 1].contiguous(), act[g:g + 1].contiguous(), r[g:g + 1].contiguous(), s2[g:g + 1].contiguous(),
                       d[g:g + 1].contiguous(), l1)
        assert_same(loss[g:g + 1], l1.cpu().numpy(), "loss of trainer %d" % g)
        for w in range(5):
            assert_same(vecs[w][g], S.get_params(w), "vector %d of trainer %d" % (w, g))
        assert S.counters() == Lg.counters()
        S.close()
    Lg.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. launches per iteration and per update do not depend on G
def launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def launch_counts(env_golden, env27_golden, shape, G, per):
    """Launches of an act pass, one lockstep iteration (act, step, commit, update) and one ring-sampled update with Ng = 8
    envs per trainer; for shapes the env cannot drive, an act pass and an explicit update of 64 rows per trainer."""
    Ng, B = 8, 64
    loss = torch.zeros(G, device=DEV)
    x = dev(np.zeros((G * B, shape[0]), np.float32))
    if shape in LOOP_ROUTES:
        city, params = short_episode_env(env_golden, env27_golden)
        pool = engine.EnvBatch(city, params, Ng, max_subgoals=64).make_scenarios(Ng, seed=5)
        env = ring_env(city, params, G * Ng, pool, 0)
        L = learner(shape, G, replay_capacity=G * 16 * Ng, lockstep_envs=G * Ng, batch_size=B, algo=algo_of("ddqn", shape))
        L.init_params(0)
        if per:
            L.per_enable_trainers()
        engine.train_run(env, L, 10, eps=0.3)                              # 80 transitions per trainer: updates run
        out = dict(act=launches(lambda: L.act(x, 0.3)),
                   iteration=launches(lambda: engine.train_run(env, L, 1, eps=0.3, want_stats=False)),
                   update=launches(lambda: L.update(loss=loss)))
        env.close()
    else:
        L = learner(shape, G, algo=algo_of("ddqn", shape))
        L.init_params(0)
        a, r = torch.zeros(G * B, dtype=torch.int32, device=DEV), torch.zeros(G * B, device=DEV)
        out = dict(act=launches(lambda: L.act(x, 0.3)), update=launches(lambda: L.update_batch(x, a, r, x, r, loss)))
    L.close()
    return out


LAUNCH_LEGS = [(s, per) for s in ROUTES for per in ((False, True) if s in LOOP_ROUTES else (False,))]


@pytest.mark.parametrize("shape,per", LAUNCH_LEGS, ids=["%s-%s" % (route_id(s), "per" if p else "uniform") for s, p in LAUNCH_LEGS])
def test_launch_count_does_not_depend_on_g(env_golden, env27_golden, shape, per):
    """DESIGN section 4: the grids' x dimension is what a stand-alone learner picks for the per-trainer size and G rides on
    gridDim.y, so G = 16 launches exactly what G = 1 launches per act pass, per lockstep iteration and per update."""
    one = launch_counts(env_golden, env27_golden, shape, 1, per)
    many = launch_counts(env_golden, env27_golden, shape, 16, per)
    assert one == many, (one, many)
    assert all(v > 0 for v in one.values()), one


# ---------------------------------------------------------------------------------------------------------------------
# 9. federation with probes drawn from the ring at one env per trainer
def test_federate_ring_probes_one_env_per_trainer(env_golden, env27_golden):
    """G = 64 trainers of one env each: federate() draws 10 probes per trainer from the ring (Philox).  They are distinct,
    trainer-local indices in range, and every round, evaluated on the rows those indices name in the trainer's own ring
    column, passes fl_restatement.check_rounds against float64."""
    G, Ng, iters = 64, 1, 30
    shape = SHIPPED[0]
    city, params = short_episode_env(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, G - 1, max_subgoals=64).make_scenarios(G - 1, seed=3)
    env = ring_env(city, params, G, pool, 0)
    L = learner(shape, G, seed=21, algo=engine.ALGO_DDQN, replay_capacity=G * 64, lockstep_envs=G)
    L.init_params(21)
    engine.train_run(env, L, iters, eps=0.5)
    n_g = L.replay_size() // G
    assert n_g == iters
    before = L.get_params(0)
    rest, counters = [L.get_params(w) for w in (1, 2, 3)], L.counters()
    idx, losses, chosen = L.federate(want_details=True)
    torch.cuda.synchronize()
    idx = idx.cpu().numpy()
    after = L.get_params(0)
    for row in idx:
        assert len(set(row.tolist())) == 10 and (row >= 0).all() and (row < n_g).all(), row
    assert len({tuple(row) for row in idx}) > 1                          # every trainer draws with its own key
    probes = np.stack([L.gather(idx[g].astype(np.int64) * G + g)[0] for g in range(G)])
    check_rounds(before, after, probes, losses.cpu().numpy(), chosen.cpu().numpy(), shape, range(G))
    for w, want in zip((1, 2, 3), rest):
        assert_same(L.get_params(w), want, "vector %d across the aggregation" % w)
    assert L.counters() == counters
    env.close(); L.close()
