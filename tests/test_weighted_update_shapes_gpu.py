"""Prioritised-replay and Huber updates at every Q-network route against float64 (qnet_restatement.f64_update): the
importance weight is_w, the |Q - y| write-back abs_err and the loss_kind branch pass through the fp32 update kernel
(learner.cu update_kernel) and the head epilogue of the tensor-core training kernel (tc_train.cu) on every route the shape
sweep pins; the integrated PER update (update() drawing from the SumTree) is pinned to its composition from the public
pieces; and the SumTree (per.cu) runs at its capacity limit, on the sampler's grid-stride path and with a total below 1."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import PER_MAX, city_and_params, dev, n_sm  # noqa: F401  (module fixture)
from qnet_restatement import abs_err_bound, draw_batch, f64_forward, f64_unpack, f64_update, net_layers
from qnet_restatement import loss_kind_reset  # noqa: F401  (fixture)
from shapes import FIXED_SHIPPED, LEGS, ROUTES, SHAPES, expected_route, shape_id
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu


VARIANTS = {                          # weighted, abs_err requested, loss kind
    "w-mse": (True, True, "mse"),
    "huber": (False, True, "huber"),
    "w-huber": (True, True, "huber"),
    "err-only": (False, True, "mse"),
    "w-noerr": (True, False, "mse"),
}


def _cases():
    out = []
    for shape in ROUTES:
        for leg in LEGS:
            if leg.endswith("-dqn"):
                algo = engine.ALGO_DQN
            else:
                algo = engine.ALGO_DUELING if shape[3] else engine.ALGO_DDQN
            marks = []
            if leg.startswith("B4096") and shape[4] != FIXED_SHIPPED and shape[:4] != (100, [64, 64], 27, 0):
                marks = [pytest.mark.skip(reason="B = 4096 takes B64-ddqn's route (32-row tiles, fused TD, NPRE = 2) on 128 CTAs; "
                                                 "it runs on the shipped shapes, which bench.py --per 1 trains at that batch")]
            for v in VARIANTS:
                out.append(pytest.param(shape, leg, algo, v, marks=marks, id="%s-%s-%s" % (shape_id(shape), leg, v)))
    return out


def test_route_table_covers_every_route():
    """ROUTES keeps one shape of every distinct route of the shape sweep's table."""
    assert {s[4] for s in SHAPES} <= {s[4] for s in ROUTES}


@pytest.mark.parametrize("shape,leg,algo,variant", _cases())
def test_weighted_update_vs_float64_and_oracle(dqn_golden, shape, leg, algo, variant, n_sm, loss_kind_reset):
    """update_batch_per, 4 updates (the hard target update at the third included), tensor cores on and off (one learner when
    the route has no tensor-core kernels), each learner against float64 at its own parameters:
      - loss within 2e-5 relative, every gradient entry within 2e-4 |g64| + 2e-5 + 2^-20 S64, S64 the sum of the magnitudes
        of the products the entry adds up (3xTF32 products carry 2^-21 relative error: this term matters only where the
        products are large and cancel, as in the V column of a dueling head, which every sample feeds);
      - EVERY |Q - y| entry (the output is prefilled with NaN, so a row no epilogue writes fails) within abs_err_bound: the act
        tests' Q bound on q_a and, through gamma, on the next-state value, plus the fp32 roundings of y and of q_a - y;
      - local and target parameters within 2e-5 of the oracle's except where Adam divides a gradient inside the fp32
        summation noise (0 < |g64| < 1e-5), or where it amplifies the measured kernel - oracle gradient difference: Adam's
        step is lr m^ / sqrt(v^), so a first-moment difference dm moves it by lr dm^ / sqrt(v^), which is large where m has
        cancelled over the steps while v has not; entries whose accumulated lr dm^ / sqrt(v^) exceeds 1e-5 (half the
        tolerance) count as noisy too.  Noisy entries: at most 4 lr, and under a quarter of the entries.
    Weights in (0, 1] with exact 1s and 0s (a zero-weight sample still reports its |Q - y|); samples on a ReLU kink, a DDQN
    next-state tie or the Huber branch point are redrawn (draw_batch), at most 5 % of a batch; with Huber at least 10 % of the
    samples lie on each branch."""
    in_dim, hidden, n_actions, dueling, route = shape
    B = LEGS[leg]
    weighted, want_err, kind = VARIANTS[variant]
    rng = np.random.default_rng([B, algo, in_dim, sum(hidden), n_actions, sorted(VARIANTS).index(variant)])
    net = O.make_net(in_dim, hidden, n_actions, dueling)
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    lr = 5e-4
    learners = []
    for tc in ((True, False) if route[0] is not None else (False,)):
        L = engine.Learner(in_dim, hidden, n_actions, dueling, algo, lr=lr, gamma=0.99, batch_size=64, update_loop=3,
                           replay_capacity=1000, loss=kind)
        assert L.set_tensor_cores(tc) == tc
        assert L.route(B) == expected_route(route, B, n_sm, tc), (tc, L.route(B))
        learners.append((tc, L))
    P = learners[0][1].P
    local0 = rng.normal(0, 0.15, P).astype(np.float32)
    target0 = rng.normal(0, 0.15, P).astype(np.float32)
    for _, L in learners:
        L.set_params(local0, 0); L.set_params(target0, 1)
    O.set_loss_kind(kind)
    OL = O.OracleLearner(net, algo, local0, update_loop=3)
    OL.target[:] = target0
    noisy = {tc: np.zeros(P, bool) for tc, _ in learners}
    dm = {tc: np.zeros(P) for tc, _ in learners}          # |m_kernel - m_oracle| carried by Adam's first moment
    drift = {tc: np.zeros(P) for tc, _ in learners}       # sum over the steps of lr dm^ / sqrt(v^)
    loss = torch.zeros(1, device="cuda")
    for step in range(4):
        locals_ = [L.get_params(0) for _, L in learners]
        targets = [L.get_params(1) for _, L in learners]
        s, a, r, s2, d, w, redrawn = draw_batch(dqn_golden, rng, layers, dueling, algo, locals_, targets[0], B, in_dim,
                                                n_actions, kind, weighted)
        assert max(redrawn.values()) <= 0.05 * B + 4, (step, redrawn)
        _, g_or, _ = OL.update(s, a, r, s2, d, is_w=np.ones(B, np.float32) if w is None else w)
        s_d, a_d, r_d, s2_d, d_d = dev(s), dev(a), dev(r), dev(s2), dev(d)
        w_d = dev(w) if weighted else None
        for (tc, L), loc, tgt in zip(learners, locals_, targets):
            l64, g64, ae64, y64, mag64 = f64_update(layers, algo, dueling, loc, tgt, s, a, r, s2, d, w, kind, abs_terms=True)
            if kind == "huber":
                assert (ae64 < 1).mean() >= 0.1 and (ae64 > 1).mean() >= 0.1, (step, tc, float((ae64 < 1).mean()))
            ae = torch.full((B,), float("nan"), device="cuda") if want_err else None
            L.update_batch_per(s_d, a_d, r_d, s2_d, d_d, w_d, ae, loss)
            torch.cuda.synchronize()
            what = (step, tc)
            assert np.isclose(float(loss), l64, rtol=2e-5, atol=0), what + (float(loss), l64)
            gg = L.get_params(4).astype(np.float64)
            gbound = 2e-4 * np.abs(g64) + 2e-5 + 2.0 ** -20 * mag64
            err = np.abs(gg - g64) - gbound
            assert (err <= 0).all(), what + (float(err.max()), int(err.argmax()), int((err > 0).sum()))
            if want_err:
                ae = ae.cpu().numpy().astype(np.float64)
                err = np.abs(ae - ae64) - abs_err_bound(y64, r, ae64)
                assert not np.isnan(ae).any(), what + (np.flatnonzero(np.isnan(ae))[:8],)
                assert (err <= 0).all(), what + (float(err.max()), int(err.argmax()), int((err > 0).sum()))
            dm[tc] = 0.9 * dm[tc] + 0.1 * np.abs(gg - g_or)
            t_adam = step + 1
            drift[tc] += lr * (dm[tc] / (1 - 0.9 ** t_adam)) / (np.sqrt(OL.v.astype(np.float64) / (1 - 0.999 ** t_adam)) + 1e-8)
            noisy[tc] |= ((np.abs(g64) < 1e-5) & (g64 != 0)) | (drift[tc] > 1e-5)
            for got, want in ((L.get_params(0), OL.local), (L.get_params(1), OL.target)):
                dp = np.abs(got - want)
                assert (dp[~noisy[tc]] <= 2e-5).all() and dp.max() <= 4 * lr, what + (float(dp[~noisy[tc]].max()), float(dp.max()))
    for tc, L in learners:
        assert noisy[tc].mean() < 0.25, (tc, noisy[tc].mean())
        L.close()


# ---------------------------------------------------------------------------------------------------------------------
# The integrated PER update: uavrl_learner_update draws its slots with the sampler's Philox stream (key seed ^ 0x9E12, counter
# the count of sampling calls), which per_sample without a tape reproduces on a twin learner.
PER_BATCHES = [64, 4096, 6000, 12000]
ALPHA, EPS_PER = 0.6, 0.01


def leaf_of(e):
    """ReplayTree.batch_update's priority of a float32 |Q - y| (fp32, as the reference computes it)."""
    e = np.float32(e) + np.float32(EPS_PER)
    return np.power(np.minimum(e, np.float32(1.0)), np.float32(ALPHA)).astype(np.float64)


def check_leaves_vs_f64(leaves, slots, ae64, y64, r, exclude):
    """The refreshed leaves of the sampled slots against min(|e64| + eps, 1)^alpha: with delta = abs_err_bound, the leaf may
    be off by alpha x_lo^(alpha - 1) delta (the largest slope of x^alpha over [x_lo, x], x_lo = max(x - delta, eps)) plus the
    fp32 roundings of |e| + eps and of powf (4 ulp).  Samples whose |e64| + eps lies within delta of the clip at 1 are not
    judged, nor are those in `exclude` (next-state ties)."""
    delta = abs_err_bound(y64, r, ae64)
    x = np.minimum(ae64 + EPS_PER, 1.0)
    want = x ** ALPHA
    x_lo = np.maximum(x - delta, EPS_PER)
    bound = ALPHA * x_lo ** (ALPHA - 1.0) * (delta + 2.0 ** -23 * x) + 2.0 ** -21 * want
    judged = ~exclude & (np.abs(ae64 + EPS_PER - 1.0) > delta)
    assert judged.mean() >= 0.9, judged.mean()
    err = np.abs(leaves[slots] - want) - bound
    assert (err[judged] <= 0).all(), (float(err[judged].max()), int(np.flatnonzero(judged)[err[judged].argmax()]))


def ddqn_ties(layers, local, s2):
    q = np.sort(f64_forward(f64_unpack(layers, local), 0, s2)[0], 1)
    return (q[:, -1] - q[:, -2]) < 1e-3


def run_composed(A, Bl, B, logical_of):
    """A: update(); Bl: per_sample -> gather -> update_batch_per -> per_set_errors(clip); logical_of maps physical slots to
    the replay's logical indices.  Parameters, Adam moments and loss must end bit-identical.  Returns the composed step's
    slots, |Q - y| and (batch, weights, parameters before the step) for judge_composed."""
    loss_a = torch.zeros(1, device="cuda"); loss_b = torch.zeros(1, device="cuda")
    local_b, target_b = Bl.get_params(0), Bl.get_params(1)
    A.update(loss=loss_a)
    slots, w = Bl.per_sample(B)
    sl = slots.cpu().numpy()
    s, a, r, s2, d = Bl.gather(logical_of(sl))
    ae = torch.full((B,), float("nan"), device="cuda")
    Bl.update_batch_per(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), w, ae, loss_b)
    Bl.per_set_errors(slots, ae, clip=True)
    torch.cuda.synchronize()
    assert float(loss_a) == float(loss_b) and np.isfinite(float(loss_a))
    for which in (0, 1, 2, 3):
        assert np.array_equal(A.get_params(which), Bl.get_params(which)), which
    return sl, ae.cpu().numpy().astype(np.float64), (s, a, r, s2, d, w.cpu().numpy(), local_b, target_b)


def assert_same_tree(A, Bl, n_slots):
    la, ta, ba = A.per_state(n_slots)
    lb, tb, bb = Bl.per_state(n_slots)
    assert np.array_equal(la, lb) and ta == tb and ba == bb
    return lb


def judge_composed(layers, algo, sl, ae, batch, leaves):
    """The composed step's |Q - y| and refreshed leaves against float64, once per distinct slot; DDQN next-state ties
    (two best local values within 1e-3: a* may differ between correct implementations) are not judged, and are few."""
    first = np.unique(sl, return_index=True)[1]
    s, a, r, s2, d = [x[first] for x in batch[:5]]
    local, target = batch[6:]
    sl, ae = sl[first], ae[first]
    _, _, ae64, y64 = f64_update(layers, algo, 0, local, target, s, a, r, s2, d)
    tie = ddqn_ties(layers, local, s2) & (d == 0) if algo != engine.ALGO_DQN else np.zeros(len(sl), bool)
    assert tie.mean() <= 0.05
    err = np.abs(ae - ae64) - abs_err_bound(y64, r, ae64)
    assert (err[~tie] <= 0).all(), float(err[~tie].max())
    check_leaves_vs_f64(leaves, sl, ae64, y64, r, tie)


@pytest.mark.parametrize("B", PER_BATCHES)
def test_per_update_is_its_composition_flat(B):
    """Flat replay (push), wrapped once, random priorities: update() with PER on equals per_sample -> gather ->
    update_batch_per -> per_set_errors(clip) bit for bit (parameters, Adam moments, loss, leaves, total, beta) over 2 steps;
    the composed step's |Q - y| and refreshed leaves match float64."""
    cap = B + B // 2 + 37
    layers = net_layers(100, [64, 64], 27, 0)
    twins = []
    for _ in range(2):
        L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B, replay_capacity=cap, seed=5, update_loop=3)
        L.init_params(0)
        L.per_enable()
        twins.append(L)
    A, Bl = twins
    rng = np.random.default_rng(B)
    pushed = 0
    for n in (cap // 2, cap // 2, cap // 3):          # the third push wraps: the oldest transition is no longer slot 0
        obs = torch.tensor(rng.standard_normal((n, 100)), dtype=torch.float32, device="cuda")
        nxt = torch.tensor(rng.standard_normal((n, 100)), dtype=torch.float32, device="cuda")
        act = torch.tensor(rng.integers(0, 27, n), dtype=torch.int32, device="cuda")
        rew = torch.tensor(rng.standard_normal(n), dtype=torch.float32, device="cuda")
        done = torch.tensor(rng.random(n) < 0.1, dtype=torch.uint8, device="cuda")
        for L in twins:
            L.push(obs, act, rew, nxt, done)
        pushed += n
    err0 = torch.tensor(rng.exponential(0.3, cap), dtype=torch.float32, device="cuda")
    for L in twins:
        L.per_set_errors(torch.arange(cap, dtype=torch.int32, device="cuda"), err0, clip=False)
    oldest = pushed % cap
    logical_of = lambda sl: (sl.astype(np.int64) - oldest) % cap      # noqa: E731
    assert_same_tree(A, Bl, cap)
    for step in range(2):
        sl, ae, batch = run_composed(A, Bl, B, logical_of)
        leaves = assert_same_tree(A, Bl, cap)
        if step == 0:
            judge_composed(layers, engine.ALGO_DDQN, sl, ae, batch, leaves)
    A.close(); Bl.close()


@pytest.mark.parametrize("B", PER_BATCHES)
def test_per_update_is_its_composition_lockstep(env_golden, env27_golden, B):
    """Lockstep ring filled by train_run(do_update=False) on two identical env / learner pairs, one leaf made dominant (half the
    total) so that one batch draws it many times: update() equals its composition bit for bit over 2 steps; the head frame (the
    one receiving the next observations) keeps priority 0 and is never drawn; the dominant slot ends with the single priority
    of its |Q - y| (every duplicate reports the same error); the composed step matches float64."""
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N, F = 1024, 16
    R = F + 1
    layers = net_layers(100, [64, 64], 27, 0)
    pairs = []
    for _ in range(2):
        env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
        env.generate_pool(512, seed=2)
        env.reset(0)
        L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B, replay_capacity=N * F, lockstep_envs=N,
                           seed=1, update_loop=3)
        L.init_params(0)
        L.per_enable()
        engine.train_run(env, L, F + 5, eps=0.5, do_update=False)
        pairs.append((env, L))
    A, Bl = pairs[0][1], pairs[1][1]
    leaves = assert_same_tree(A, Bl, N * R).reshape(R, N)
    head = np.flatnonzero((leaves == 0).all(1))
    assert len(head) == 1 and A.replay_size() == N * F
    head = int(head[0])
    oldest = (head + 1) % R
    logical_of = lambda sl: ((sl // N - oldest) % R) * N + sl % N      # noqa: E731
    dom = ((head + 3) % R) * N + 17
    for L in (A, Bl):
        L.per_set_priorities(torch.tensor([dom], dtype=torch.int32, device="cuda"),
                             torch.tensor([leaves.sum()], dtype=torch.float64, device="cuda"))
    for step in range(2):
        sl, ae, batch = run_composed(A, Bl, B, logical_of)
        lv = assert_same_tree(A, Bl, N * R)
        assert not (sl // N == head).any() and (lv.reshape(R, N)[head] == 0).all()
        if step == 0:
            hits = sl == dom
            assert hits.sum() >= B // 4, int(hits.sum())
            assert (ae[hits] == ae[hits][0]).all()
            assert np.isclose(lv[dom], leaf_of(ae[hits][0]), rtol=2.0 ** -22, atol=0)      # fp32 powf: 4 ulp
            judge_composed(layers, engine.ALGO_DDQN, sl, ae, batch, lv)
    for env, L in pairs:
        env.close(); L.close()


# ---------------------------------------------------------------------------------------------------------------------
# The SumTree at its edges


def test_per_max_capacity_vs_oracle(n_sm):
    """4 194 304 slots with dyadic priorities (every partial sum exact), 1 % of them 0: stratified draws from a tape pick
    exactly the oracle's leaves, weights within 2e-6 relative, beta as the oracle's -- B = 4096 and B = 12 000, the latter
    more draws than the sampler grid's 8 x (4 x SMs) warps (per_sample_kernel's grid-stride loop)."""
    cap = PER_MAX
    L = engine.Learner(4, [32], 5, False, engine.ALGO_DQN, batch_size=64, replay_capacity=cap, seed=5)
    L.per_enable()
    rng = np.random.default_rng(7)
    x = torch.zeros((cap, 4), dtype=torch.float32, device="cuda")
    L.push(x, torch.zeros(cap, dtype=torch.int32, device="cuda"), torch.zeros(cap, device="cuda"), x,
           torch.zeros(cap, dtype=torch.uint8, device="cuda"))
    prio = np.ldexp(rng.integers(1, 4096, cap).astype(np.float64), -10)
    prio[rng.integers(0, cap, cap // 100)] = 0.0
    L.per_set_priorities(torch.arange(cap, dtype=torch.int32, device="cuda"), torch.tensor(prio, device="cuda"))
    per = O.OraclePer(cap)
    per.add(prio)
    leaves, total, _ = L.per_state(cap)
    assert np.array_equal(leaves, prio) and total == prio.sum() == per.total
    for B in (4096, 12000):
        u = rng.random(B)
        idx_o, w_o, beta_o = per.sample(u)
        slots, w = L.per_sample(B, torch.tensor(u, device="cuda"))
        assert np.array_equal(slots.cpu().numpy().astype(np.int64) + cap - 1, idx_o), B
        np.testing.assert_allclose(w.cpu().numpy(), w_o, rtol=2e-6)
        assert L.per_state(cap)[2] == beta_o
    assert 12000 > 8 * 4 * n_sm
    L.close()


def test_per_capacity_over_limit_is_refused():
    """One slot more than the limit: per_enable refuses before it allocates or enables anything."""
    L = engine.Learner(4, [32], 5, False, engine.ALGO_DQN, batch_size=64, replay_capacity=PER_MAX + 1, seed=5)
    with pytest.raises(engine.UavrlError, match="at most 4194304 slots"):
        L.per_enable()
    with pytest.raises(engine.UavrlError, match="not enabled"):
        L.per_state(1)
    L.close()


@pytest.mark.parametrize("cap", [16, 12])
def test_per_total_below_one(cap):
    """Nine fresh transitions at priority 0.01^0.6 ~ 0.063 sum to 0.57 and batch 8 draws: SumTree.total() is int(tree[0]) = 0
    (replay_buffer.py:120-121), so every segment is [0, 0], every draw walks to the leftmost leaf (slot 0 of a power-of-two
    ring, slot rot = 4 of the 12-slot one, whose leaf order is rotated), prob = p / 0 is infinite, every raw weight
    (n prob)^-beta is 0 and the normalised weights 0 / 0 are NaN.  The reference does exactly this with numpy float64 scalars
    and arrays: it emits RuntimeWarnings (divide by zero, invalid value) and raises nothing, so its weights are all NaN.  The
    device matches the oracle leaf for leaf and NaN for NaN, and the integrated update that weighs the loss with them reports
    a NaN loss, as a weighted loss with the reference's weights would."""
    L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=8, replay_capacity=cap, seed=5, update_loop=3)
    L.init_params(0)
    L.per_enable()
    per = O.OraclePer(cap)
    rng = np.random.default_rng(cap)
    n = 9
    x = torch.tensor(rng.standard_normal((n, 100)), dtype=torch.float32, device="cuda")
    L.push(x, torch.tensor(rng.integers(0, 27, n), dtype=torch.int32, device="cuda"),
           torch.tensor(rng.standard_normal(n), dtype=torch.float32, device="cuda"), x,
           torch.zeros(n, dtype=torch.uint8, device="cuda"))
    per.push(np.zeros(n, np.float32))
    leaves, total, _ = L.per_state(cap)
    assert np.array_equal(leaves, per.leaves()) and 0.5 < total < 1
    u = rng.random(8)
    with np.errstate(all="ignore"):
        idx_o, w_o, beta_o = per.sample(u)
    slots, w = L.per_sample(8, torch.tensor(u, device="cuda"))
    sl = slots.cpu().numpy().astype(np.int64)
    assert np.array_equal(sl + cap - 1, idx_o)
    pow2 = 1 << (cap - 1).bit_length()
    assert (sl == pow2 - cap).all()
    np.testing.assert_array_equal(w.cpu().numpy(), w_o.astype(np.float32))
    assert np.isnan(w_o).all() and L.per_state(cap)[2] == beta_o
    loss = torch.zeros(1, device="cuda")
    L.update(loss=loss)
    torch.cuda.synchronize()
    assert np.isnan(float(loss))
    L.close()
