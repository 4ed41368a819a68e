"""Q-network shapes beyond the shipped ones (input 100, hidden [64, 64] / [64] / [128, 64], 27 actions) against a float64
reference: every row of shapes.SHAPES, with the route it must take pinned through Learner.route, so every kernel variant is
compared by value here and a shape that silently moves to another route fails."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import dev, n_sm  # noqa: F401  (module fixture)
from qnet_restatement import big_inputs, f64_forward, f64_unpack, f64_update, near_relu_kink, net_layers
from shapes import SHAPES, SHIPPED, act_sizes, expected_route, shape_id
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu


def rup(x, m):
    return -(-x // m) * m


def test_table_covers_every_route():
    """The table keeps at least one shape of every route, and none of the shipped shapes (other tests cover those)."""
    assert not [s for s in SHAPES if (s[0], s[1], s[2], s[3]) in SHIPPED]
    has = lambda pred: any(pred(*s) for s in SHAPES)                                                  # noqa: E731
    assert has(lambda i, h, a, d, r: r[0] == "generic" and r[1] == "generic"), "generic forward + generic training"
    assert has(lambda i, h, a, d, r: r[0] == "fixed" and r[1] == "fixed"), "FIXED forward + FIXED training"
    assert has(lambda i, h, a, d, r: r[0] == "generic" and any(rup(w, 16) % 32 == 16 for w in h)), "16-column tail"
    assert has(lambda i, h, a, d, r: r[0] is not None and r[1] is None), "tensor-core TD feeding the fp32 update"
    assert has(lambda i, h, a, d, r: r[0] is None), "fp32 only"
    assert has(lambda i, h, a, d, r: len(h) == 4 and r[1] is not None), "4 hidden layers on the training kernel"
    for i, h, a, d, r in SHAPES:
        if any(rup(w, 16) % 32 == 16 for w in h) and r[0] is not None:
            assert r[0] == "generic", "a 16-column chunk has no FIXED chain"


UPDATE_LEGS = {                        # B, algo: fused TD with NPRE = 1 / 2, fused TD with 64-row tiles, separate TD passes
    "B64-dqn": (64, engine.ALGO_DQN),
    "B64-ddqn": (64, engine.ALGO_DDQN),
    "B6000-ddqn": (6000, engine.ALGO_DDQN),
    "B12000-dqn": (12000, engine.ALGO_DQN),
}


def make_learner(shape, algo=engine.ALGO_DQN):
    in_dim, hidden, n_actions, dueling, _ = shape
    L = engine.Learner(in_dim, hidden, n_actions, dueling, algo, lr=5e-4, gamma=0.99, batch_size=64, update_loop=3,
                       replay_capacity=1000)
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    assert L.P == sum(o * i + o for o, i in layers) == O.net_param_count(O.make_net(in_dim, hidden, n_actions, dueling))
    return L, layers


@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
def test_route_is_pinned(shape, n_sm):
    L, _ = make_learner(shape)
    ns = act_sizes(shape[4], n_sm) + [b for b, _ in UPDATE_LEGS.values()]
    for tc in (True, False):
        assert L.set_tensor_cores(tc) == (tc and shape[4][0] is not None)
        for n in ns:
            assert L.route(n) == expected_route(shape[4], n, n_sm, tc), (shape_id(shape), tc, n)
    L.close()


@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
def test_act_vs_float64(dqn_golden, shape, n_sm):
    """Q of the act pass (eps-greedy tapes) with the tensor cores on and off within 2e-5 abs + 2e-5 rel of float64; greedy
    actions identical wherever the float64 top-2 gap exceeds 1e-4, random ones equal to the tape; both as the oracle acts."""
    in_dim, hidden, n_actions, dueling, route = shape
    rng = np.random.default_rng(in_dim * 1000 + sum(hidden) + n_actions)
    net = O.make_net(in_dim, hidden, n_actions, dueling)
    L, layers = make_learner(shape)
    params = rng.normal(0, 0.15, L.P).astype(np.float32)
    L.set_params(params, 0)
    P64 = f64_unpack(layers, params)
    eps = 0.25
    for n in act_sizes(route, n_sm):
        x = big_inputs(dqn_golden, n, rng, in_dim)
        u = rng.uniform(size=n).astype(np.float32); ra = rng.integers(0, n_actions, n).astype(np.int32)
        q64 = f64_forward(P64, dueling, x)[0]
        top2 = np.sort(q64, 1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 1e-4
        assert clear.mean() >= 0.99, (n, clear.mean())
        rand = u <= eps
        a_or, q_or = O.act(net, params, x, eps, u, ra)
        assert (np.abs(q_or - q64) <= 2e-5 + 2e-5 * np.abs(q64)).all()
        for tc in (True, False):
            assert L.set_tensor_cores(tc) == (tc and route[0] is not None)
            assert L.route(n) == expected_route(route, n, n_sm, tc)
            a, q = L.act(dev(x), eps, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
            a, q = a.cpu().numpy(), q.cpu().numpy()
            err = np.abs(q - q64) - (2e-5 + 2e-5 * np.abs(q64))
            assert (err <= 0).all(), (n, tc, float(err.max()), np.unravel_index(err.argmax(), err.shape))
            assert np.array_equal(a[rand], ra[rand]), (n, tc)
            greedy = ~rand & clear
            assert np.array_equal(a[greedy], q64[greedy].argmax(1)), (n, tc, int((a[greedy] != q64[greedy].argmax(1)).sum()))
            assert np.array_equal(a[rand | clear], a_or[rand | clear]), (n, tc)
    L.close()


@pytest.mark.parametrize("leg", list(UPDATE_LEGS))
@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
def test_update_vs_float64_and_oracle(dqn_golden, shape, leg, n_sm):
    """4 updates on explicit batches (the hard target update at epoch 3 included): loss within 2e-5 relative of float64 and
    the oracle, every gradient entry within 2e-4 |g64| + 2e-5 of float64, local and target parameters within 2e-5 of the
    oracle's except where Adam divides a gradient inside the fp32 summation noise (0 < |g64| < 1e-5: at most 4 lr, and under
    a quarter of the entries).  An exactly zero float64 gradient (a unit dead over the whole batch, an action no sample took)
    is not noise: those parameters are held to 2e-5 as well."""
    in_dim, hidden, n_actions, dueling, route = shape
    B, algo = UPDATE_LEGS[leg]
    rng = np.random.default_rng(B + algo + in_dim * 1000 + sum(hidden) + n_actions)
    net = O.make_net(in_dim, hidden, n_actions, dueling)
    L, layers = make_learner(shape, algo)
    assert L.set_tensor_cores(True) == (route[0] is not None)
    assert L.route(B) == expected_route(route, B, n_sm)
    local0 = rng.normal(0, 0.15, L.P).astype(np.float32)
    target0 = rng.normal(0, 0.15, L.P).astype(np.float32)
    L.set_params(local0, 0); L.set_params(target0, 1)
    OL = O.OracleLearner(net, algo, local0, update_loop=3)
    OL.target[:] = target0
    lr = 5e-4
    loss = torch.zeros(1, device="cuda")
    noisy = np.zeros(L.P, bool)
    for step in range(4):
        s = big_inputs(dqn_golden, B, rng, in_dim); s2 = big_inputs(dqn_golden, B, rng, in_dim)
        # a sample whose hidden pre-activation lies within fp32 noise of 0 may take the other side of the ReLU in any fp32-grade
        # evaluation and then moves that unit's gradient row by its whole term: such rows are drawn again
        P64 = f64_unpack(layers, L.get_params(0))
        for _ in range(20):
            kink = near_relu_kink(P64, dueling, s)
            if not kink.any():
                break
            s[kink] = big_inputs(dqn_golden, int(kink.sum()), rng, in_dim)
        assert not kink.any()
        a = rng.integers(0, n_actions, B).astype(np.int32)
        r = rng.normal(0, 1.0, B).astype(np.float32)
        d = (rng.uniform(size=B) < 0.1).astype(np.float32)
        if algo != engine.ALGO_DQN:
            # where the two best local next-state values tie within the arithmetic noise two correct implementations may
            # pick different a*: such samples are marked terminal (as test_tc_update_large_batch_vs_oracle does)
            ql = np.sort(O.net_forward(net, L.get_params(0), s2).astype(np.float64), 1)
            d[(ql[:, -1] - ql[:, -2]) < 1e-3] = 1.0
        l64, g64 = f64_update(layers, algo, dueling, L.get_params(0), L.get_params(1), s, a, r, s2, d)[:2]
        L.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), loss)
        lo, _ = OL.update(s, a, r, s2, d)
        torch.cuda.synchronize()
        assert np.isclose(float(loss), l64, rtol=2e-5, atol=0), (step, float(loss), l64)
        assert np.isclose(float(loss), lo, rtol=2e-5, atol=0), (step, float(loss), lo)
        gg = L.get_params(4).astype(np.float64)
        err = np.abs(gg - g64) - (2e-4 * np.abs(g64) + 2e-5)
        assert (err <= 0).all(), (step, float(err.max()), int(err.argmax()), int((err > 0).sum()))
        noisy |= (np.abs(g64) < 1e-5) & (g64 != 0)
        for got, want in ((L.get_params(0), OL.local), (L.get_params(1), OL.target)):
            dp = np.abs(got - want)
            assert (dp[~noisy] <= 2e-5).all() and dp.max() <= 4 * lr, (step, float(dp[~noisy].max()), float(dp.max()))
    assert noisy.mean() < 0.25, noisy.mean()
    L.close()


def test_vanet5_is_rejected():
    """VAnet5 at hiden_dim 64 ([128, 64, 64, 64], dueling): the fp32 update kernel would need 245 760 B of shared memory
    (over the 227 KB a block may use), so the learner refuses it at creation."""
    hidden = engine.NET_KINDS["VAnet5"][0](64)
    assert hidden == [128, 64, 64, 64] and engine.NET_KINDS["VAnet5"][1] == 1
    with pytest.raises(engine.UavrlError, match="network too large for the shared-memory resident kernels"):
        engine.Learner(100, hidden, 27, True, engine.ALGO_DDQN)
