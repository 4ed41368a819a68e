"""Data-parallel forms of the Q-network update at every route of the shape sweep, on one GPU.

The data-parallel update runs the single-GPU kernels with the loss scaled by 1/global_batch instead of 1/B, and takes its
optimiser step either in reduce_adam_kernel (compute_grads: apply = 0, then apply_grads: nparts = 0) or in
dp_allreduce_adam_kernel (update_dp, train_run_dp).  This file pins:
  a. world = 1: update, compute_grads + apply_grads and update_dp give the same bits at every route, both loss kinds, tensor
     cores on and off (parameters, Adam moments, loss, counters, weight images);
  b. global_batch != B: the two data-parallel forms agree bit for bit and match float64 scaled by B / global_batch;
  c. W ranks simulated in one process (compute_grads per shard, float32 sum in rank order, apply_grads) against float64 and
     the oracle on the concatenated batch;
  d. prioritised replay: the partials-only path refreshes the SumTree exactly as the plain update does;
  e. train_run_dp against train_run, and against its composition from train_run + compute_grads + apply_grads;
  f. the refusals of train_run_dp, train_profile, compute_grads and update_dp, which leave every state untouched."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import city_and_params
from test_qnet_shapes_gpu import expected_route, shape_id
from test_tc_gpu import big_inputs, dev, net_layers
from test_weighted_f64_cpu import draw_batch, f64_update_w
from test_weighted_update_shapes_gpu import FIXED_SHIPPED, LEGS, ROUTES
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

SHIPPED = next(s for s in ROUTES if s[:4] == (100, [64, 64], 27, 0))
GENERIC = next(s for s in ROUTES if s[4][0] == "generic" and s[4][1] == "generic")
FP32 = next(s for s in ROUTES if s[4][0] is None)
KINDS = ("mse", "huber")
LR = 5e-4


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def loss_kind_reset():
    yield
    O.set_loss_kind("mse")            # the oracle's loss kind is process-wide state


def algo_of(leg, dueling):
    """The sweep's convention: "-dqn" legs run DQN, the others double DQN (the dueling trainer on a dueling head)."""
    if leg.endswith("-dqn"):
        return engine.ALGO_DQN
    return engine.ALGO_DUELING if dueling else engine.ALGO_DDQN


def tc_settings(route):
    return (True, False) if route[0] is not None else (False,)


def make(shape, algo, B, cap, kind="mse", tc=True, **kw):
    in_dim, hidden, n_actions, dueling, _ = shape
    L = engine.Learner(in_dim, hidden, n_actions, dueling, algo, lr=LR, gamma=0.99, batch_size=B, update_loop=3,
                       replay_capacity=cap, loss=kind, **kw)
    assert L.set_tensor_cores(tc) == tc
    return L


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def assert_same_learner(A, X, what):
    """Parameters, target and Adam moments bit for bit; the reduced gradient equal as values (dp_allreduce_adam_kernel stores
    0.f + g, which turns a -0 into +0 and nothing else); counters equal."""
    for which in (0, 1, 2, 3):
        assert np.array_equal(bits(A.get_params(which)), bits(X.get_params(which))), what + (which,)
    ga, gx = A.get_params(4), X.get_params(4)
    assert np.array_equal(ga, gx), what + ("grad", int((ga != gx).sum()))
    assert ((bits(ga) == bits(gx)) | (ga == 0)).all(), what
    assert A.counters() == X.counters(), what + (A.counters(), X.counters())


def assert_same_images(learners, in_dim, rng, what):
    """The fp32 and tensor-core weight images the optimiser step refreshes: a probe batch through the act kernel on every
    arithmetic path the learners have gives identical Q values and actions."""
    obs = torch.tensor(rng.uniform(-1, 1, size=(256, in_dim)).astype(np.float32), device="cuda")
    for tc in (True, False):
        on = [L.set_tensor_cores(tc) for L in learners]
        assert len(set(on)) == 1
        if tc and not on[0]:
            continue
        out = [L.act(obs, 0.3, want_q=True) for L in learners]
        for a, q in out[1:]:
            assert torch.equal(out[0][0], a) and torch.equal(out[0][1], q), what + (tc,)


def push(L, s, a, r, s2, d):
    L.push(dev(s), dev(a.astype(np.int32)), dev(r.astype(np.float32)), dev(s2), dev(d.astype(np.uint8)))


# ---------------------------------------------------------------------------------------------------------------------
# a. world = 1: update == compute_grads + apply_grads == update_dp, bit for bit
A_LEGS = ["B64-dqn", "B64-ddqn", "B6000-ddqn", "B12000-dqn"]


def _a_cases():
    return [pytest.param(shape, leg, kind, id="%s-%s-%s" % (shape_id(shape), leg, kind))
            for shape in ROUTES for leg in A_LEGS for kind in KINDS]


@pytest.mark.parametrize("shape,leg,kind", _a_cases())
def test_world1_forms_are_bit_identical(dqn_golden, shape, leg, kind, n_sm):
    """Three learners with the same parameters, replay and index tapes: A runs update, B compute_grads(B) + apply_grads, C
    connect_self + update_dp(B).  Five updates with update_loop 3 (the hard target update at the third; both parities of
    C's receive buffer) end every step in the same parameters, target, Adam moments, gradient (up to the sign of a zero),
    loss and counters, and the weight images give the same Q values on a probe batch."""
    in_dim, hidden, n_actions, dueling, route = shape
    B = LEGS[leg]
    algo = algo_of(leg, dueling)
    rng = np.random.default_rng([B, algo, in_dim, sum(hidden), n_actions, KINDS.index(kind)])
    cap = B + B // 2 + 37
    s, s2 = big_inputs(dqn_golden, cap, rng, in_dim), big_inputs(dqn_golden, cap, rng, in_dim)
    a = rng.integers(0, n_actions, cap); r = rng.normal(0, 1.0, cap); d = rng.uniform(size=cap) < 0.1
    for tc in tc_settings(route):
        trio = [make(shape, algo, B, cap, kind, tc) for _ in range(3)]
        A, Bl, C = trio
        assert A.route(B) == expected_route(route, B, n_sm, tc), (tc, A.route(B))
        local0 = rng.normal(0, 0.15, A.P).astype(np.float32)
        target0 = rng.normal(0, 0.15, A.P).astype(np.float32)
        for L in trio:
            L.set_params(local0, 0); L.set_params(target0, 1)
            push(L, s, a, r, s2, d)
        C.connect_self()
        losses = [torch.zeros(1, device="cuda") for _ in range(3)]
        for step in range(5):
            idx = dev(rng.permutation(cap)[:B].astype(np.int32))
            A.update(idx_tape=idx, loss=losses[0])
            Bl.compute_grads(B, idx_tape=idx, loss=losses[1])
            Bl.apply_grads()
            C.update_dp(B, idx_tape=idx, loss=losses[2])
            torch.cuda.synchronize()
            what = (tc, step)
            lv = [float(x) for x in losses]
            assert np.isfinite(lv[0]) and lv[0] == lv[1] == lv[2], what + tuple(lv)
            assert A.counters() == (step + 1, step + 1)
            assert np.array_equal(bits(A.get_params(4)), bits(Bl.get_params(4))), what
            assert_same_learner(A, Bl, what)
            assert_same_learner(A, C, what)
        assert not np.array_equal(A.get_params(1), target0)
        assert_same_images(trio, in_dim, rng, (tc,))
        for L in trio:
            L.close()


# ---------------------------------------------------------------------------------------------------------------------
# b. global_batch != B at world = 1
GB_B = 64


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", ROUTES, ids=shape_id)
def test_global_batch_scaling_vs_float64(dqn_golden, shape, kind, n_sm):
    """B = 64 local samples, global_batch 2B and 3B + 5 in turn over 4 updates (the hard target update at the third),
    tensor cores on and off: update_dp(gb) equals compute_grads(gb) + apply_grads bit for bit, the loss share is
    (B / gb) x the float64 batch loss within 2e-5 relative, and every gradient entry lies within (B / gb) (2e-4 |g64| + 2e-5
    + 2^-20 S64) of (B / gb) g64 (S64: the summed magnitudes of the products the entry adds up, as in the weighted sweep)."""
    in_dim, hidden, n_actions, dueling, route = shape
    B = GB_B
    algo = engine.ALGO_DUELING if dueling else engine.ALGO_DDQN
    rng = np.random.default_rng([in_dim, sum(hidden), n_actions, KINDS.index(kind), 7])
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    idx = dev(np.arange(B, dtype=np.int32))
    for tc in tc_settings(route):
        pair = [make(shape, algo, B, B + 1, kind, tc) for _ in range(2)]
        Bl, C = pair
        assert Bl.route(B) == expected_route(route, B, n_sm, tc)
        local0 = rng.normal(0, 0.15, Bl.P).astype(np.float32)
        target0 = rng.normal(0, 0.15, Bl.P).astype(np.float32)
        for L in pair:
            L.set_params(local0, 0); L.set_params(target0, 1)
        C.connect_self()
        lb, lc = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
        for step, gb in enumerate((2 * B, 3 * B + 5, 2 * B, 3 * B + 5)):
            local, target = Bl.get_params(0), Bl.get_params(1)
            s, a, r, s2, d, _, redrawn = draw_batch(dqn_golden, rng, layers, dueling, algo, [local], target, B, in_dim,
                                                    n_actions, kind, False)
            assert max(redrawn.values()) <= 0.05 * B + 4, (step, redrawn)
            l64, g64, _, _, mag64 = f64_update_w(layers, algo, dueling, local, target, s, a, r, s2, d, None, kind, abs_terms=True)
            for L in pair:                      # B transitions, then one dummy: capacity B + 1, logical index i = slot i
                push(L, s, a, r, s2, d)
                push(L, s[:1], a[:1], r[:1], s2[:1], d[:1])
            Bl.compute_grads(gb, idx_tape=idx, loss=lb)
            Bl.apply_grads()
            C.update_dp(gb, idx_tape=idx, loss=lc)
            torch.cuda.synchronize()
            what = (tc, step, gb)
            assert float(lb) == float(lc), what + (float(lb), float(lc))
            assert_same_learner(Bl, C, what)
            k = B / gb
            assert np.isclose(float(lb), k * l64, rtol=2e-5, atol=0), what + (float(lb), k * l64)
            gg = Bl.get_params(4).astype(np.float64)
            err = np.abs(gg - k * g64) - k * (2e-4 * np.abs(g64) + 2e-5 + 2.0 ** -20 * mag64)
            assert (err <= 0).all(), what + (float(err.max()), int(err.argmax()), int((err > 0).sum()))
        for L in pair:
            L.close()


# ---------------------------------------------------------------------------------------------------------------------
# c. W ranks simulated in one process against float64 and the oracle on the concatenated batch
C_ALGO = {37: "ddqn", 64: "dqn", 6000: "ddqn", 12000: "dqn"}      # per-rank B: two tiles with a ragged one, NPRE, 64-row, split TD


def _c_cases():
    out = []
    for shape in ROUTES:
        for B in C_ALGO:
            for kind in KINDS:
                out.append(pytest.param(shape, 2, B, kind, id="%s-W2-B%d-%s" % (shape_id(shape), B, kind)))
    for shape in (SHIPPED, GENERIC, FP32):
        for W in (3, 8):
            for B in (37, 64):
                for kind in KINDS:
                    out.append(pytest.param(shape, W, B, kind, id="%s-W%d-B%d-%s" % (shape_id(shape), W, B, kind)))
    return out


@pytest.mark.parametrize("shape,W,B,kind", _c_cases())
def test_simulated_allreduce_vs_float64_and_oracle(dqn_golden, shape, W, B, kind, n_sm, loss_kind_reset):
    """W learners with the same parameters; each step draws a W B batch against the float64 networks (draw_batch: no sample
    on a ReLU kink, a DDQN next-state tie or the Huber branch point), learner r holds shard r (plus one dummy transition) and
    runs compute_grads(W B, idx_tape = 0..B-1); the W gradients are summed in rank order in float32 and copied into every
    learner, then apply_grads.  Over 4 steps (the hard target update at the third):
      - the W loss shares sum to the float64 full-batch loss within 2e-5 relative;
      - every entry of the summed gradient lies within 2e-4 |g64| + 2e-5 + 2^-20 S64 of the float64 full-batch gradient;
      - local and target parameters lie within 2e-5 of the oracle's on the concatenated batch, but for the weighted sweep's
        noisy entries (0 < |g64| < 1e-5, or an accumulated Adam amplification lr dm^ / sqrt(v^) of the measured
        kernel - oracle gradient difference above 1e-5): those within 4 lr, and under a quarter of the entries;
      - the W replicas stay bit-identical."""
    in_dim, hidden, n_actions, dueling, route = shape
    algo = algo_of(C_ALGO[B], dueling)
    rng = np.random.default_rng([W, B, algo, in_dim, sum(hidden), n_actions, KINDS.index(kind)])
    net = O.make_net(in_dim, hidden, n_actions, dueling)
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    ranks = [make(shape, algo, B, B + 1, kind, route[0] is not None) for _ in range(W)]
    assert ranks[0].route(B) == expected_route(route, B, n_sm, route[0] is not None), ranks[0].route(B)
    P = ranks[0].P
    local0 = rng.normal(0, 0.15, P).astype(np.float32)
    target0 = rng.normal(0, 0.15, P).astype(np.float32)
    for L in ranks:
        L.set_params(local0, 0); L.set_params(target0, 1)
    O.set_loss_kind(kind)
    OL = O.OracleLearner(net, algo, local0, update_loop=3)
    OL.target[:] = target0
    idx = dev(np.arange(B, dtype=np.int32))
    losses = [torch.zeros(1, device="cuda") for _ in range(W)]
    noisy, dm, drift = np.zeros(P, bool), np.zeros(P), np.zeros(P)
    n = W * B
    for step in range(4):
        local, target = ranks[0].get_params(0), ranks[0].get_params(1)
        s, a, r, s2, d, _, redrawn = draw_batch(dqn_golden, rng, layers, dueling, algo, [local], target, n, in_dim, n_actions,
                                                kind, False)
        assert max(redrawn.values()) <= 0.05 * n + 4, (step, redrawn)
        l64, g64, _, _, mag64 = f64_update_w(layers, algo, dueling, local, target, s, a, r, s2, d, None, kind, abs_terms=True)
        _, g_or, _ = OL.update(s, a, r, s2, d, is_w=np.ones(n, np.float32))
        for q, L in enumerate(ranks):
            sh = slice(q * B, (q + 1) * B)
            push(L, s[sh], a[sh], r[sh], s2[sh], d[sh])
            push(L, s[:1], a[:1], r[:1], s2[:1], d[:1])
            L.compute_grads(n, idx_tape=idx, loss=losses[q])
        grads = [L.grad_tensor() for L in ranks]
        total = grads[0].clone()
        for g in grads[1:]:
            total += g
        for g in grads:
            g.copy_(total)
        for L in ranks:
            L.apply_grads()
        torch.cuda.synchronize()
        what = (step,)
        share = sum(float(x) for x in losses)
        assert np.isclose(share, l64, rtol=2e-5, atol=0), what + (share, l64)
        gg = total.cpu().numpy().astype(np.float64)
        err = np.abs(gg - g64) - (2e-4 * np.abs(g64) + 2e-5 + 2.0 ** -20 * mag64)
        assert (err <= 0).all(), what + (float(err.max()), int(err.argmax()), int((err > 0).sum()))
        for L in ranks[1:]:
            for which in (0, 1, 2, 3, 4):
                assert np.array_equal(bits(ranks[0].get_params(which)), bits(L.get_params(which))), what + (which,)
            assert L.counters() == ranks[0].counters() == (step + 1, step + 1)
        dm = 0.9 * dm + 0.1 * np.abs(gg - g_or)
        t_adam = step + 1
        drift += LR * (dm / (1 - 0.9 ** t_adam)) / (np.sqrt(OL.v.astype(np.float64) / (1 - 0.999 ** t_adam)) + 1e-8)
        noisy |= ((np.abs(g64) < 1e-5) & (g64 != 0)) | (drift > 1e-5)
        for got, want in ((ranks[0].get_params(0), OL.local), (ranks[0].get_params(1), OL.target)):
            dp = np.abs(got - want)
            assert (dp[~noisy] <= 2e-5).all() and dp.max() <= 4 * LR, what + (float(dp[~noisy].max()), float(dp.max()))
    assert noisy.mean() < 0.25, noisy.mean()
    for L in ranks:
        L.close()


# ---------------------------------------------------------------------------------------------------------------------
# d. prioritised replay: the SumTree draws the batch, and every form refreshes it the same way
@pytest.mark.parametrize("B", [64, 4096])
@pytest.mark.parametrize("shape", [SHIPPED, GENERIC, FP32], ids=shape_id)
def test_per_forms_are_bit_identical(dqn_golden, shape, B, n_sm):
    """A (update), B (compute_grads + apply_grads) and C (connect_self + update_dp) with prioritised replay on, the same seed
    and no index tape, over a wrapped flat replay with random priorities: after each of 5 steps the parameters, Adam moments,
    loss, counters and the SumTree (leaves, total, beta) are identical."""
    in_dim, hidden, n_actions, dueling, route = shape
    algo = engine.ALGO_DUELING if dueling else engine.ALGO_DDQN
    rng = np.random.default_rng([B, in_dim, sum(hidden), 11])
    cap = B + B // 2 + 37
    trio = [make(shape, algo, B, cap, tc=route[0] is not None, seed=5) for _ in range(3)]
    A, Bl, C = trio
    assert A.route(B) == expected_route(route, B, n_sm, route[0] is not None)
    local0 = rng.normal(0, 0.15, A.P).astype(np.float32)
    target0 = rng.normal(0, 0.15, A.P).astype(np.float32)
    for L in trio:
        L.set_params(local0, 0); L.set_params(target0, 1)
        L.per_enable()
    for m in (cap // 2, cap // 2, cap // 3):         # the third push wraps
        s, s2 = big_inputs(dqn_golden, m, rng, in_dim), big_inputs(dqn_golden, m, rng, in_dim)
        a = rng.integers(0, n_actions, m); r = rng.normal(0, 1.0, m); d = rng.uniform(size=m) < 0.1
        for L in trio:
            push(L, s, a, r, s2, d)
    err0 = torch.tensor(rng.exponential(0.3, cap), dtype=torch.float32, device="cuda")
    for L in trio:
        L.per_set_errors(torch.arange(cap, dtype=torch.int32, device="cuda"), err0, clip=False)
    C.connect_self()
    losses = [torch.zeros(1, device="cuda") for _ in range(3)]
    leaves0 = A.per_state(cap)[0]
    for step in range(5):
        A.update(loss=losses[0])
        Bl.compute_grads(B, loss=losses[1])
        Bl.apply_grads()
        C.update_dp(B, loss=losses[2])
        torch.cuda.synchronize()
        lv = [float(x) for x in losses]
        assert np.isfinite(lv[0]) and lv[0] == lv[1] == lv[2], (step,) + tuple(lv)
        assert_same_learner(A, Bl, (step,))
        assert_same_learner(A, C, (step,))
        la, ta, ba = A.per_state(cap)
        for X in (Bl, C):
            lx, tx, bx = X.per_state(cap)
            assert np.array_equal(la, lx) and ta == tx and ba == bx, step
    assert not np.array_equal(la, leaves0)
    for L in trio:
        L.close()


# ---------------------------------------------------------------------------------------------------------------------
# e. train_run_dp, the loop bench.py times for every data-parallel headline
T_DP = 60
# name: (N envs, batch_size, hidden, dueling, algo, tensor cores, PER, uavrl_set_pdl, uavrl_set_fuse_td)
E_LEGS = {
    "N1024-ddqn": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, True, False, 1, 1),       # 32-row tiles, fused TD
    "N1024-dqn": (1024, 1024, [64, 64], 0, engine.ALGO_DQN, True, False, 1, 1),
    "N1024-dueling": (1024, 1024, [64], 1, engine.ALGO_DUELING, True, False, 1, 1),
    "N6144-ddqn": (6144, 6144, [64, 64], 0, engine.ALGO_DDQN, True, False, 1, 1),       # 64-row tiles, fused TD
    "N2048-B12000-dqn": (2048, 12000, [64, 64], 0, engine.ALGO_DQN, True, False, 1, 1),  # separate TD passes
    "N1024-ddqn-fp32": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, False, False, 1, 1),
    "N1024-ddqn-per": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, True, True, 1, 1),
    "N1024-ddqn-pdl0-fuse0": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, True, False, 0, 0),
    "N1024-ddqn-pdl0-fuse1": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, True, False, 0, 1),
    "N1024-ddqn-pdl1-fuse0": (1024, 1024, [64, 64], 0, engine.ALGO_DDQN, True, False, 1, 0),
}


@pytest.fixture(scope="module")
def scenarios(env_golden, env27_golden):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, 64, max_subgoals=64)
    sc = env.make_scenarios(1024, seed=8)
    env.close()
    return city, params, sc


@pytest.fixture
def schedule_reset():
    yield
    _lib.lib().uavrl_set_pdl(1)                 # library defaults: PDL on, fused TD on
    _lib.lib().uavrl_set_fuse_td(1)


def lockstep_pair(scenarios, N, B, hidden, dueling, algo, tc=True, per=False, frames=16, in_dim=100, **kw):
    city, params, sc = scenarios
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    L = engine.Learner(in_dim, hidden, 27, dueling, algo, batch_size=B, replay_capacity=N * frames, lockstep_envs=N, seed=1,
                       update_loop=3, **kw)
    L.init_params(0)
    assert L.set_tensor_cores(tc) == tc
    if per:
        L.per_enable()
    return env, L


def snapshot(env, L):
    torch.cuda.synchronize()
    out = dict(("p%d" % w, bits(L.get_params(w))) for w in range(5))
    out["counters"] = L.counters()
    n = L.replay_size()
    out["replay_size"] = n
    if n:
        for k, x in zip(("s", "a", "r", "s2", "d"), L.gather(np.arange(n))):
            out[k] = x.view(np.uint32) if x.dtype == np.float32 else x
    for k, x in env.get_state().items():
        out["env_" + k] = np.asarray(x)
    return out


def assert_same_snapshot(a, b, grad_pm0=True):
    assert a.keys() == b.keys()
    for k in a:
        if k == "p4" and grad_pm0:                  # the dp kernel's gradient is 0.f + g
            ga, gb = a[k].view(np.float32), b[k].view(np.float32)
            assert np.array_equal(ga, gb) and ((a[k] == b[k]) | (ga == 0)).all(), k
        elif isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
        else:
            assert a[k] == b[k], (k, a[k], b[k])


@pytest.mark.parametrize("leg", list(E_LEGS))
def test_train_run_dp_equals_train_run(scenarios, leg, n_sm, schedule_reset):
    """Two identical env + lockstep learner pairs, warmed up without updates; T = 60 iterations of train_run (one update per
    iteration) on the first and of train_run_dp(global_batch = batch_size) after connect_self on the second end in the same
    parameters, target, Adam moments, gradient (up to the sign of a zero), counters, replay contents, env state and, with
    prioritised replay, SumTree."""
    N, B, hidden, dueling, algo, tc, per, pdl, fuse = E_LEGS[leg]
    _lib.lib().uavrl_set_pdl(pdl)
    _lib.lib().uavrl_set_fuse_td(fuse)
    frames = 8 if N >= 6144 else 16
    warm = B // N + 2
    pairs = [lockstep_pair(scenarios, N, B, hidden, dueling, algo, tc, per, frames) for _ in range(2)]
    (e1, L1), (e2, L2) = pairs
    route = FIXED_SHIPPED if tc else (None, None, False, False, True)
    want = expected_route(route, B, n_sm, tc)
    if not fuse:
        want["td_fused"] = False
    assert L1.route(B) == want, L1.route(B)
    L2.connect_self()
    for env, L in pairs:
        engine.train_run(env, L, warm, eps=1.0, do_update=False)
        assert L.replay_size() > B and L.counters() == (0, 0)
    p_warm = L1.get_params(0)
    st = engine.train_run(e1, L1, T_DP, 0.2, updates_per_iter=1)
    assert st.updates == T_DP
    engine.train_run_dp(e2, L2, T_DP, 0.2, global_batch=B)
    a, b = snapshot(e1, L1), snapshot(e2, L2)
    assert a["counters"] == (T_DP, T_DP)
    assert_same_snapshot(a, b)
    p = L1.get_params(0)
    assert np.isfinite(p).all() and not np.array_equal(p, p_warm)
    if per:
        n = N * (frames + 1)
        l1, t1, b1 = L1.per_state(n)
        l2, t2, b2 = L2.per_state(n)
        assert np.array_equal(l1, l2) and t1 == t2 and b1 == b2
    for env, L in pairs:
        env.close(); L.close()


def test_train_run_dp_global_batch_is_its_composition(scenarios, n_sm):
    """train_run_dp(T, global_batch = 3 batch_size) equals T rounds of train_run(1, do_update = False) + compute_grads(3 batch)
    + apply_grads, bit for bit (parameters, counters, replay, env state)."""
    N = B = 1024
    pairs = [lockstep_pair(scenarios, N, B, [64, 64], 0, engine.ALGO_DDQN) for _ in range(2)]
    (e1, L1), (e2, L2) = pairs
    L2.connect_self()
    for env, L in pairs:
        engine.train_run(env, L, 3, eps=1.0, do_update=False)
    for _ in range(T_DP):
        engine.train_run(e1, L1, 1, 0.2, do_update=False, want_stats=False)
        L1.compute_grads(3 * B)
        L1.apply_grads()
    engine.train_run_dp(e2, L2, T_DP, 0.2, global_batch=3 * B)
    a, b = snapshot(e1, L1), snapshot(e2, L2)
    assert a["counters"] == (T_DP, T_DP)
    assert_same_snapshot(a, b)
    for env, L in pairs:
        env.close(); L.close()


# ---------------------------------------------------------------------------------------------------------------------
# f. refusals: refused with their error code before anything is enqueued, and nothing changes
def assert_refused(call, code, match, states):
    """call() raises UavrlError with `code` and a message matching `match`, launches no kernel, and every (env, learner)
    in `states` keeps its parameters, counters, replay and env state."""
    before = [snapshot(env, L) for env, L in states]
    n0 = _lib.launch_count()
    with pytest.raises(engine.UavrlError, match=r"uavrl error %d: .*%s" % (code, match)):
        call()
    assert _lib.launch_count() == n0
    for (env, L), b in zip(states, before):
        assert_same_snapshot(b, snapshot(env, L), grad_pm0=False)


ERR_INVALID, ERR_STATE = -1, -3
R_N = 64


def refusal_case(scenarios, case):
    """(env, learner, call, code, message) of one refused train_run_dp call."""
    B, warm, kw, connect = 64, 3, {}, True
    if case == "grouped":
        kw, connect = dict(trainers=2), False
    elif case == "cold-ring":
        B, warm = 256, 2                           # 128 transitions, 192 after the first iteration's commit: <= 256
    elif case == "lockstep-mismatch":
        kw, warm = dict(lockstep_envs=R_N // 2), 0
    elif case.startswith("in_dim"):
        kw, warm = dict(in_dim=int(case.split("-")[1])), 0
    elif case == "not-connected":
        connect = False
    if "lockstep_envs" in kw:
        city, params, sc = scenarios
        env = engine.EnvBatch(city, params, R_N, max_subgoals=64, auto_reset=True)
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        env.reset(0)
        L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B, replay_capacity=R_N * 16, seed=1, **kw)
        L.init_params(0)
    else:
        env, L = lockstep_pair(scenarios, R_N, B, [64, 64], 0, engine.ALGO_DDQN, **kw)
    if connect:
        L.connect_self()
    if warm:
        engine.train_run(env, L, warm, eps=1.0, do_update=False)
    gb = {"gb0": 0, "gb-neg": -B}.get(case, B)
    expect = {
        "not-connected": (ERR_STATE, "before uavrl_learner_comm_connect"),
        "grouped": (ERR_INVALID, "several trainers"),
        "gb0": (ERR_INVALID, "bad argument"),
        "gb-neg": (ERR_INVALID, "bad argument"),
        "lockstep-mismatch": (ERR_INVALID, "lockstep_envs must equal env.n_envs"),
        "in_dim-64": (ERR_INVALID, "in_dim must be 100"),
        "in_dim-128": (ERR_INVALID, "in_dim must be 100"),
        "cold-ring": (ERR_STATE, "replay holds <= batch_size transitions"),
    }[case]
    return env, L, (lambda: engine.train_run_dp(env, L, 5, 0.2, gb)), expect


@pytest.mark.parametrize("case", ["not-connected", "grouped", "gb0", "gb-neg", "lockstep-mismatch", "in_dim-64", "in_dim-128",
                                  "cold-ring"])
def test_train_run_dp_refusals(scenarios, case):
    """train_run_dp refuses, before it launches anything and leaving env, ring, parameters and counters as they were: a learner
    not connected, a grouped learner, global_batch <= 0, lockstep_envs != env.n, a learner whose in_dim is not the 100-float
    observation (the env step writes 100-float rows into the ring), and a ring that would hold <= batch_size transitions at
    the first update (every rank must take part in every exchange)."""
    env, L, call, (code, match) = refusal_case(scenarios, case)
    assert_refused(call, code, match, [(env, L)])
    env.close(); L.close()


@pytest.mark.parametrize("in_dim", [64, 128])
def test_train_profile_refuses_in_dim(scenarios, in_dim):
    """train_profile refuses a learner whose in_dim is not 100 before anything else, with train_run's message."""
    env, L = lockstep_pair(scenarios, R_N, 64, [64, 64], 0, engine.ALGO_DDQN, in_dim=in_dim)
    assert_refused(lambda: engine.train_profile(env, L, 2, 0.2), ERR_INVALID, "in_dim must be 100", [(env, L)])
    env.close(); L.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("call", ["train_run_dp", "train_profile"])
def test_device_mismatch_is_refused(scenarios, call):
    """An env on device 0 and a learner on device 1: refused with train_run's message, nothing launched."""
    city, params, sc = scenarios
    env = engine.EnvBatch(city, params, R_N, max_subgoals=64, auto_reset=True)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=R_N * 16, lockstep_envs=R_N,
                       seed=1, device=1)
    if call == "train_run_dp":
        L.connect_self()
        fn = lambda: engine.train_run_dp(env, L, 5, 0.2, 64)         # noqa: E731
    else:
        fn = lambda: engine.train_profile(env, L, 2, 0.2)            # noqa: E731
    n0 = _lib.launch_count()
    with pytest.raises(engine.UavrlError, match="uavrl error -1: env and learner live on different devices"):
        fn()
    assert _lib.launch_count() == n0 and L.counters() == (0, 0) and L.replay_size() == 0
    env.close(); L.close()


def test_compute_grads_and_update_dp_refuse_cold_replay(dqn_golden):
    """compute_grads and update_dp on a replay holding exactly batch_size transitions: refused with UAVRL_ERR_STATE before the
    epoch counts, so a data-parallel rank that retries stays on the other ranks' sample keys and target schedule.  One more
    transition and both run, at epoch 1."""
    B = 64
    rng = np.random.default_rng(3)
    shape = SHIPPED
    pair = [make(shape, engine.ALGO_DDQN, B, 4 * B) for _ in range(2)]
    Bl, C = pair
    C.connect_self()
    s, s2 = big_inputs(dqn_golden, B + 1, rng), big_inputs(dqn_golden, B + 1, rng)
    a = rng.integers(0, 27, B + 1); r = rng.normal(0, 1.0, B + 1); d = rng.uniform(size=B + 1) < 0.1
    for L in pair:
        L.init_params(0)
        push(L, s[:B], a[:B], r[:B], s2[:B], d[:B])
    params = [L.get_params(0) for L in pair]
    for L, fn in ((Bl, lambda: Bl.compute_grads(B)), (C, lambda: C.update_dp(B))):
        for _ in range(2):                                          # a retry is refused the same way
            n0 = _lib.launch_count()
            with pytest.raises(engine.UavrlError, match="uavrl error -3: replay holds <= batch_size transitions"):
                fn()
            assert _lib.launch_count() == n0 and L.counters() == (0, 0) and L.replay_size() == B
    for L, p in zip(pair, params):
        assert np.array_equal(L.get_params(0), p)
        push(L, s[B:], a[B:], r[B:], s2[B:], d[B:])
    Bl.compute_grads(B)
    Bl.apply_grads()
    C.update_dp(B)
    torch.cuda.synchronize()
    assert Bl.counters() == C.counters() == (1, 1)
    assert_same_learner(Bl, C, ())
    for L in pair:
        L.close()
