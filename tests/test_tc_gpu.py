"""Tensor-core (wgmma, 3xTF32) forward path vs the fp32 CUDA-core path and the oracle: same actions,
Q within 2e-5, and the full update (TD targets from the tensor-core pass) inside the reference-trainer
tolerances for every algorithm; also large ragged batches and the explicit switch."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import dev
from qnet_restatement import big_inputs, f64_update, net_layers

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("hidden,dueling", [([64, 64], 0), ([64], 1), ([64], 0), ([128, 64], 1)])
def test_tc_act_matches_fp32_path_and_oracle(dqn_golden, hidden, dueling):
    from uavrl_b200 import engine
    g = dqn_golden
    rng = np.random.default_rng(3)
    net = O.make_net(100, hidden, 27, dueling)
    P = O.net_param_count(net)
    params = rng.normal(0, 0.15, P).astype(np.float32)
    n = 5000                                              # ragged: 39 full tiles of 128 + 8
    x = np.tile(np.concatenate([g["batch_s"].reshape(-1, 100), g["batch_s2"].reshape(-1, 100)]), (4, 1))[:n]
    x = x + rng.normal(0, 0.01, x.shape).astype(np.float32)
    L = engine.Learner(100, hidden, 27, dueling, 1)
    L.set_params(params, 0)
    on = L.set_tensor_cores(True)
    if hidden == [128, 64]:
        assert not on                                     # does not fit the SMEM-resident kernel: fp32 path serves it
        L.close()
        return
    assert on
    u = rng.uniform(size=n).astype(np.float32); ra = rng.integers(0, 27, n).astype(np.int32)
    a_tc, q_tc = L.act(dev(x), 0.2, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
    assert not L.set_tensor_cores(False)
    a_32, q_32 = L.act(dev(x), 0.2, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
    a_or, q_or = O.act(net, params, x, 0.2, u, ra)
    q_tc, q_32 = q_tc.cpu().numpy(), q_32.cpu().numpy()
    np.testing.assert_allclose(q_tc, q_or, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(q_32, q_or, rtol=2e-5, atol=2e-5)
    # actions: identical except where the top-2 Q gap is inside the arithmetic noise (none expected at this scale)
    top2 = np.sort(q_or, 1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-4
    assert clear.mean() > 0.99
    assert np.array_equal(a_tc.cpu().numpy()[clear], a_or[clear])
    assert np.array_equal(a_32.cpu().numpy()[clear], a_or[clear])
    L.close()


CASES = {"dueling_vanet2": ([64], 1, 2), "ddqn_qvalue3": ([64, 64], 0, 1), "dqn_qvalue3": ([64, 64], 0, 0), "dqn_qnet2": ([64], 0, 0)}


@pytest.mark.parametrize("name", list(CASES))
def test_tc_td_targets_keep_update_parity(dqn_golden, name):
    """The learner tests run with the tensor-core path on by default; this one pins it explicitly and
    compares TC-on vs TC-off trajectories of 10 updates."""
    from uavrl_b200 import engine
    g = dqn_golden
    hidden, dueling, algo = CASES[name]
    out = {}
    for tc in (True, False):
        L = engine.Learner(100, hidden, 27, dueling, algo, batch_size=64, update_loop=3, replay_capacity=1000)
        assert L.set_tensor_cores(tc) == tc
        L.set_params(g[name + "_local0"], 0); L.set_params(g[name + "_target0"], 1)
        loss = torch.zeros(1, device="cuda"); losses = []
        for step in range(10):
            L.update_batch(dev(g["batch_s"][step]), dev(g["batch_a"][step], torch.int32), dev(g["batch_r"][step]),
                           dev(g["batch_s2"][step]), dev(g["batch_d"][step]), loss)
            losses.append(float(loss))
        out[tc] = (np.array(losses), L.get_params(0), L.get_params(1))
        L.close()
    np.testing.assert_allclose(out[True][0], g[name + "_loss"], rtol=2e-5)
    np.testing.assert_allclose(out[True][0], out[False][0], rtol=1e-5)
    np.testing.assert_allclose(out[True][1], g[name + "_local"][-1], atol=2e-5)
    np.testing.assert_allclose(out[True][1], out[False][1], atol=5e-6)
    np.testing.assert_allclose(out[True][2], out[False][2], atol=5e-6)


# ---------------------------------------------------------------------------------------------------------------------
# The tile variants the large BASELINE configs select (launch_tc_forward: R = 64 rows per tile from n >= 64 x 132,
# R = 128 from n >= 128 x 132 when 128-row tiles fit shared memory; tc_train: R = 64 from B >= 32 x 132) compared with the oracle by VALUE, ragged last tiles.
@pytest.mark.parametrize("n", [12000, 20011])
@pytest.mark.parametrize("hidden,dueling", [([64, 64], 0), ([64], 1)])
def test_tc_act_large_tiles_vs_oracle(dqn_golden, n, hidden, dueling):
    from uavrl_b200 import engine
    rng = np.random.default_rng(n)
    net = O.make_net(100, hidden, 27, dueling)
    params = rng.normal(0, 0.15, O.net_param_count(net)).astype(np.float32)
    x = big_inputs(dqn_golden, n, rng)
    u = rng.uniform(size=n).astype(np.float32); ra = rng.integers(0, 27, n).astype(np.int32)
    L = engine.Learner(100, hidden, 27, dueling, 1)
    L.set_params(params, 0)
    assert L.set_tensor_cores(True)
    a_tc, q_tc = L.act(dev(x), 0.25, u_tape=dev(u), rand_tape=dev(ra), want_q=True)
    a_or, q_or = O.act(net, params, x, 0.25, u, ra)
    np.testing.assert_allclose(q_tc.cpu().numpy(), q_or, rtol=2e-5, atol=2e-5)
    top2 = np.sort(q_or, 1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-4
    assert clear.mean() > 0.99
    assert np.array_equal(a_tc.cpu().numpy()[clear], a_or[clear])
    L.close()


@pytest.mark.parametrize("B", [12000, 20011])
@pytest.mark.parametrize("name", ["dqn_qvalue3", "ddqn_qvalue3", "dueling_vanet2"])
def test_tc_update_large_batch_vs_oracle(dqn_golden, name, B):
    """Trainer.update on an explicit batch of 12 000 / 20 011 transitions (TD-target passes with R = 64 / 128 rows per tile,
    training chain R = 64, 94 / 157 weight-gradient chunks).  At this batch size two fp32 implementations differ by their
    summation order alone (the oracle adds 20 000 per-sample terms one after the other per thread; the kernels add 128-sample
    tensor-core partials), so a float64 numpy restatement arbitrates: the CUDA gradient (fp32 accumulation in the tensor cores, then a fixed-order
    fp32 sum of the partials) must match float64 within 2e-4 relative / 2e-5 absolute on EVERY entry; against the oracle 99.9 % of the entries meet the same bound and none is off by more than 2e-4.  Parameters after each of 4 updates (incl. the
    hard update at epoch 3): within 2e-5 of the oracle's except where Adam divides a gradient that is itself inside the fp32
    summation noise (|g| < 1e-5: the step is +-lr whichever way the noise points), and never further than 4 lr."""
    from uavrl_b200 import engine
    g = dqn_golden
    hidden, dueling, algo = CASES[name]
    rng = np.random.default_rng(B + algo)
    net = O.make_net(100, hidden, 27, dueling)
    L = engine.Learner(100, hidden, 27, dueling, algo, lr=5e-4, gamma=0.99, batch_size=64, update_loop=3, replay_capacity=1000)
    assert L.set_tensor_cores(True)
    L.set_params(g[name + "_local0"], 0); L.set_params(g[name + "_target0"], 1)
    OL = O.OracleLearner(net, algo, g[name + "_local0"], update_loop=3)
    OL.target[:] = g[name + "_target0"]
    layers = net_layers(100, hidden, 27, dueling)
    loss = torch.zeros(1, device="cuda")
    noisy = np.zeros(L.P, bool)
    for step in range(4):
        s = big_inputs(g, B, rng); s2 = big_inputs(g, B, rng)
        a = rng.integers(0, 27, B).astype(np.int32)
        r = rng.normal(0, 1.0, B).astype(np.float32)
        d = (rng.uniform(size=B) < 0.1).astype(np.float32)
        if algo != 0:
            # double-DQN selects a* = argmax_a q_local(s') and gathers q_target(s', a*): where the two best local values tie to
            # within the arithmetic noise, two correct implementations may pick different a* and then disagree by a whole
            # q_target gap on that sample.  Such samples are marked terminal (the next-state value is multiplied by 0).
            ql = np.sort(O.net_forward(net, L.get_params(0), s2).astype(np.float64), 1)
            d[(ql[:, -1] - ql[:, -2]) < 1e-3] = 1.0
        l64, g64 = f64_update(layers, algo, dueling, L.get_params(0), L.get_params(1), s, a, r, s2, d)[:2]
        L.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), loss)
        lo, grads = OL.update(s, a, r, s2, d)
        torch.cuda.synchronize()
        assert np.isclose(float(loss), lo, rtol=2e-5), (step, float(loss), lo)
        assert np.isclose(float(loss), l64, rtol=2e-5), (step, float(loss), l64)
        gg = L.get_params(4).astype(np.float64)
        bound = 2e-4 * np.abs(g64) + 2e-5
        err_gpu, err_or = np.abs(gg - g64), np.abs(grads - g64)
        assert (err_gpu <= bound).all(), (step, float((err_gpu - bound).max()))
        # (the oracle accumulates in double but evaluates the networks in fp32: it differs from float64 where a ReLU input is
        # within fp32 noise of 0, by that unit's whole contribution)
        assert err_or.max() <= 2e-4 and err_or.mean() <= 1e-6
        vs_or = np.abs(gg - grads)
        assert (vs_or <= 2e-4 * np.abs(grads) + 2e-5).mean() >= 0.999 and vs_or.max() <= 2e-4
        noisy |= np.abs(g64) < 1e-5
        dp = np.abs(L.get_params(0) - OL.local)
        assert (dp[~noisy] <= 2e-5).all() and dp.max() <= 4 * 5e-4, (step, float(dp[~noisy].max()), float(dp.max()))
        dt = np.abs(L.get_params(1) - OL.target)
        assert (dt[~noisy] <= 2e-5).all() and dt.max() <= 4 * 5e-4
    assert noisy.mean() < 0.25
    L.close()
