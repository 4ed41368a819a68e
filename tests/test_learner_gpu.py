"""CUDA learner (Q-net forward, eps-greedy, replay, TD update, Adam, hard update) through the C ABI
against (1) golden vectors produced by the reference's own trainer classes on torch CPU fp32 and
(2) the CPU oracle.  Tolerance: fp32 results within 2e-5 (abs, parameters) / 2e-4 (rel, gradients
and losses whose magnitude is ~1e3); integer outputs (actions) exact."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import dev

pytestmark = pytest.mark.gpu

CASES = {"dueling_vanet2": ([64], 1, 2), "dueling_vanet3": ([128, 64], 1, 2),
         "ddqn_qvalue3": ([64, 64], 0, 1), "dqn_qvalue3": ([64, 64], 0, 0), "dqn_qnet2": ([64], 0, 0)}


@pytest.mark.parametrize("name", list(CASES))
def test_update_matches_reference_trainers(dqn_golden, name):
    from uavrl_b200 import engine
    g = dqn_golden
    hidden, dueling, algo = CASES[name]
    L = engine.Learner(100, hidden, 27, dueling, algo, lr=5e-4, gamma=0.99, batch_size=64, update_loop=3,
                       replay_capacity=1000)
    assert L.P == g[name + "_local0"].size
    L.set_params(g[name + "_local0"], 0)
    L.set_params(g[name + "_target0"], 1)
    snap = list(g[name + "_snap"])
    loss = torch.zeros(1, device="cuda")
    for step in range(g["batch_s"].shape[0]):
        L.update_batch(dev(g["batch_s"][step]), dev(g["batch_a"][step], torch.int32), dev(g["batch_r"][step]),
                       dev(g["batch_s2"][step]), dev(g["batch_d"][step]), loss)
        torch.cuda.synchronize()
        assert np.isclose(float(loss), g[name + "_loss"][step], rtol=2e-5), (step, float(loss))
        if step in snap:
            k = snap.index(step)
            np.testing.assert_allclose(L.get_params(4), g[name + "_grads"][k], rtol=2e-4, atol=2e-4)
            np.testing.assert_allclose(L.get_params(0), g[name + "_local"][k], rtol=0, atol=2e-5)
            np.testing.assert_allclose(L.get_params(1), g[name + "_target"][k], rtol=0, atol=2e-5)
    assert L.counters() == (10, 10)
    # forward + greedy action on the final network (Trainer.get_action with eps = 0)
    a, q = L.act(dev(g["batch_s"][0]), eps=0.0, want_q=True)
    np.testing.assert_allclose(q.cpu().numpy(), g[name + "_q_final"], rtol=2e-5, atol=2e-5)
    assert np.array_equal(a.cpu().numpy(), g[name + "_q_final"].argmax(1))
    L.close()


def test_eps_greedy_tapes_vs_oracle(dqn_golden):
    from uavrl_b200 import engine
    g = dqn_golden
    rng = np.random.default_rng(0)
    for hidden, dueling in (([64, 64], 0), ([64], 1)):
        net = O.make_net(100, hidden, 27, dueling)
        P = O.net_param_count(net)
        params = rng.normal(0, 0.1, P).astype(np.float32)
        n = 1000                                   # ragged: not a multiple of the 32-sample tile
        x = np.concatenate([g["batch_s"].reshape(-1, 100), g["batch_s2"].reshape(-1, 100)])[:n]
        u = rng.uniform(size=n).astype(np.float32)
        ra = rng.integers(0, 27, n).astype(np.int32)
        L = engine.Learner(100, hidden, 27, dueling, 1)
        L.set_params(params, 0)
        for eps, train in ((0.3, 1), (1.0, 1), (0.0, 1), (0.9, 0)):
            a_ref, q_ref = O.act(net, params, x, eps, u, ra, is_train=train)
            a, q = L.act(dev(x), eps, is_train=train, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
            np.testing.assert_allclose(q.cpu().numpy(), q_ref, rtol=2e-5, atol=2e-5)
            assert np.array_equal(a.cpu().numpy(), a_ref)
        # Philox path: valid actions, ~eps fraction random
        a = L.act(dev(x), 0.5).cpu().numpy()
        assert a.min() >= 0 and a.max() < 27
        greedy = O.act(net, params, x, 0.0, u, ra)[0]
        frac = (a != greedy).mean()
        assert 0.35 < frac < 0.6                  # eps * (1 - 1/27) ~ 0.48
        L.close()


def test_replay_fifo_and_sampled_update_vs_oracle(dqn_golden):
    """ReplayMemory.add FIFO over capacity + update on injected sample indices vs the oracle."""
    from uavrl_b200 import engine
    g = dqn_golden
    cap, B = 300, 64
    s = g["batch_s"].reshape(-1, 100); s2 = g["batch_s2"].reshape(-1, 100)
    a = g["batch_a"].reshape(-1); r = g["batch_r"].reshape(-1); d = g["batch_d"].reshape(-1)
    n_all = s.shape[0]                              # 640 transitions through a 300-slot ring
    net = O.make_net(100, [64, 64], 27, 0)
    L = engine.Learner(100, [64, 64], 27, False, 1, batch_size=B, replay_capacity=cap, update_loop=2)
    p0 = g["ddqn_qvalue3_local0"]
    L.set_params(p0, 0); L.set_params(g["ddqn_qvalue3_target0"], 1)
    OL = O.OracleLearner(net, O.ALGO_DDQN, p0, update_loop=2)
    OL.target[:] = g["ddqn_qvalue3_target0"]
    rng = np.random.default_rng(1)
    pushed = 0
    loss = torch.zeros(1, device="cuda")
    for chunk in (50, 14, 100, 200, 37, 239):       # ragged pushes, wraps the ring twice
        sl = slice(pushed, pushed + chunk)
        L.push(dev(s[sl]), dev(a[sl], torch.int32), dev(r[sl]), dev(s2[sl]), dev(d[sl], torch.uint8))
        pushed += chunk
        size = min(pushed, cap)
        assert L.replay_size() == size
        # logical index j = j-th oldest stored transition
        first = pushed - size
        gs, ga, gr, gs2, gd = L.gather(np.arange(size))
        assert np.array_equal(gs, s[first:pushed]) and np.array_equal(gs2, s2[first:pushed])
        assert np.array_equal(ga, a[first:pushed]) and np.array_equal(gr, r[first:pushed])
        assert np.array_equal(gd, d[first:pushed].astype(np.uint8))
        if size <= B:
            L.update()                               # not enough data: epoch counts, nothing changes
            OL.epoch += 1
            continue
        idx = rng.permutation(size)[:B].astype(np.int32)      # random.sample: distinct indices
        L.update(idx_tape=dev(idx), loss=loss)
        lo, _ = OL.update(s[first + idx], a[first + idx], r[first + idx], s2[first + idx], d[first + idx])
        torch.cuda.synchronize()
        assert np.isclose(float(loss), lo, rtol=2e-5)
        np.testing.assert_allclose(L.get_params(0), OL.local, rtol=0, atol=2e-5)
        np.testing.assert_allclose(L.get_params(1), OL.target, rtol=0, atol=2e-5)
    assert pushed == n_all
    assert L.counters()[0] == OL.epoch
    L.close()


def test_philox_sampling_is_without_replacement(dqn_golden):
    """Batch_Size == replay size - 1: a sample without replacement then covers all but one transition.
    Rewards encode the index, the bias gradient of a 1-action net reveals which were drawn."""
    from uavrl_b200 import engine
    M, B = 257, 256
    L = engine.Learner(100, [64], 1, False, 0, batch_size=B, replay_capacity=M, update_loop=1000, gamma=0.0, lr=0.0)
    L.set_params(np.zeros(L.P, np.float32), 0); L.set_params(np.zeros(L.P, np.float32), 1)
    z = torch.zeros((M, 100), device="cuda")
    r = torch.arange(M, device="cuda", dtype=torch.float32) + 1.0      # y = r ; Q = 0 -> diff = -r
    L.push(z, torch.zeros(M, dtype=torch.int32, device="cuda"), r, z, torch.ones(M, dtype=torch.uint8, device="cuda"))
    seen = set()
    for _ in range(5):
        loss = torch.zeros(1, device="cuda")
        L.update(loss=loss)
        gb = L.get_params(4)[-1]                       # d loss / d bias = -2/B * sum(r_sampled)
        ssum = -gb * B / 2.0
        missing = round(M * (M + 1) / 2 - ssum)        # exactly one index absent iff all distinct
        assert 1 <= missing <= M, missing
        assert abs((M * (M + 1) / 2 - ssum) - missing) < 0.05
        sq = float(loss) * B                           # sum r^2 over the sample
        assert abs(sq - (M * (M + 1) * (2 * M + 1) / 6 - missing ** 2)) < 1e-3 * sq
        seen.add(missing)
    assert len(seen) >= 3                              # different draws each epoch
    L.close()


def test_data_parallel_split_equals_fused_update(dqn_golden):
    """compute_grads + apply_grads (the path a gradient all-reduce sits between) == update."""
    from uavrl_b200 import engine
    g = dqn_golden
    s = g["batch_s"].reshape(-1, 100)[:200]; s2 = g["batch_s2"].reshape(-1, 100)[:200]
    a = g["batch_a"].reshape(-1)[:200]; r = g["batch_r"].reshape(-1)[:200]; d = g["batch_d"].reshape(-1)[:200]
    Ls = []
    for _ in range(2):
        L = engine.Learner(100, [64, 64], 27, False, 1, batch_size=64, replay_capacity=200)
        L.set_params(g["ddqn_qvalue3_local0"], 0); L.set_params(g["ddqn_qvalue3_target0"], 1)
        L.push(dev(s), dev(a, torch.int32), dev(r), dev(s2), dev(d, torch.uint8))
        Ls.append(L)
    idx = dev(np.random.default_rng(2).permutation(200)[:64].astype(np.int32))
    for _ in range(3):
        Ls[0].update(idx_tape=idx)
        Ls[1].compute_grads(64, idx_tape=idx)
        gt = Ls[1].grad_tensor()
        assert gt.shape[0] == Ls[1].P and torch.isfinite(gt).all()
        Ls[1].apply_grads()
    assert np.array_equal(Ls[0].get_params(0), Ls[1].get_params(0))
    assert np.array_equal(Ls[0].get_params(1), Ls[1].get_params(1))
    for L in Ls:
        L.close()


@pytest.mark.parametrize("tc", [True, False])
def test_huber_loss_option_vs_oracle(dqn_golden, tc):
    """loss_kind = 1 (Huber / SmoothL1Loss(beta = 1), an option beside the reference's MSE): tensor-core and fp32 paths
    against the oracle, whose Huber form is pinned to torch autograd (tests/test_oracle_golden.py)."""
    from uavrl_b200 import engine
    g = dqn_golden
    name = "ddqn_qvalue3"
    net = O.make_net(100, [64, 64], 27, 0)
    L = engine.Learner(100, [64, 64], 27, False, 1, lr=5e-4, gamma=0.99, batch_size=64, update_loop=3, replay_capacity=1000, loss="huber")
    assert L.set_tensor_cores(tc) == tc
    L.set_params(g[name + "_local0"], 0); L.set_params(g[name + "_target0"], 1)
    O.set_loss_kind("huber")
    try:
        OL = O.OracleLearner(net, 1, g[name + "_local0"], update_loop=3)
        OL.target[:] = g[name + "_target0"]
        loss = torch.zeros(1, device="cuda")
        for step in range(6):
            r = g["batch_r"][step] * 3.0                          # part of the batch beyond |Q - y| = 1: the linear branch
            L.update_batch(dev(g["batch_s"][step]), dev(g["batch_a"][step], torch.int32), dev(r), dev(g["batch_s2"][step]),
                           dev(g["batch_d"][step]), loss)
            lo, grads = OL.update(g["batch_s"][step], g["batch_a"][step], r, g["batch_s2"][step], g["batch_d"][step])
            torch.cuda.synchronize()
            assert np.isclose(float(loss), lo, rtol=2e-5), (step, float(loss), lo)
            np.testing.assert_allclose(L.get_params(4), grads, rtol=2e-4, atol=2e-6)
            np.testing.assert_allclose(L.get_params(0), OL.local, rtol=0, atol=2e-5)
    finally:
        O.set_loss_kind("mse")
    L.close()
