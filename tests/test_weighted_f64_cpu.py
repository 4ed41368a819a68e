"""The float64 restatement of the Q-network update (qnet_restatement.f64_update, with importance weights and both loss kinds),
pinned before it judges any kernel: against torch autograd on the same float64 network (to 1e-12) and against the CPU
oracle's weighted update (ora_dqn_update_per under both loss kinds, at the fp32 bounds test_tc_update_large_batch_vs_oracle
uses), on the batches draw_batch builds for the GPU sweeps."""
import numpy as np
import pytest
import torch

import oracle as O
from qnet_restatement import GAMMA, abs_err_bound, draw_batch, f64_update, f64_unpack, net_layers
from qnet_restatement import loss_kind_reset  # noqa: F401  (fixture)


def torch_update(layers, algo, dueling, local, target, s, a, r, s2, d, w, loss_kind, gamma=GAMMA):
    """The same loss through torch.nn.functional in float64 and its gradient by autograd (state_dict order)."""
    def params(flat, grad):
        out = [(torch.tensor(W, requires_grad=grad), torch.tensor(b, requires_grad=grad)) for W, b in f64_unpack(layers, flat)]
        return out

    def fwd(P, x):
        h = x
        nt = len(P) - (2 if dueling else 1)
        for W, b in P[:nt]:
            h = torch.relu(h @ W.T + b)
        if dueling:
            A = h @ P[nt][0].T + P[nt][1]; V = h @ P[nt + 1][0].T + P[nt + 1][1]
            return V + A - A.mean(1, keepdim=True)
        return h @ P[nt][0].T + P[nt][1]
    PL, PT = params(local, True), params(target, False)
    s, s2 = torch.tensor(s, dtype=torch.float64), torch.tensor(s2, dtype=torch.float64)
    r, d = torch.tensor(r, dtype=torch.float64), torch.tensor(d, dtype=torch.float64)
    a = torch.tensor(a, dtype=torch.int64)
    with torch.no_grad():
        qt = fwd(PT, s2)
        nq = qt.max(1).values if algo == 0 else qt.gather(1, fwd(PL, s2).argmax(1, keepdim=True)).squeeze(1)
        y = r + gamma * nq * (1.0 - d)
    qa = fwd(PL, s).gather(1, a[:, None]).squeeze(1)
    if loss_kind == "mse":
        per = torch.nn.functional.mse_loss(qa, y, reduction="none")
    else:
        per = torch.nn.functional.smooth_l1_loss(qa, y, reduction="none", beta=1.0)
    wt = torch.ones_like(per) if w is None else torch.tensor(w, dtype=torch.float64)
    loss = (wt * per).mean()
    loss.backward()
    grad = torch.cat([t.grad.reshape(-1) for W, b in PL for t in (W, b)])
    return float(loss.detach()), grad.numpy()


CASES = {                            # (in_dim, hidden, n_actions, dueling, algo)
    "qvalue3-dqn": (100, [64, 64], 27, 0, O.ALGO_DQN),
    "qvalue3-ddqn": (100, [64, 64], 27, 0, O.ALGO_DDQN),
    "vanet2-dueling": (100, [64], 27, 1, O.ALGO_DUELING),
    "vanet3-dueling": (100, [128, 64], 27, 1, O.ALGO_DUELING),
}
VARIANTS = {"w-mse": (True, "mse"), "mse": (False, "mse"), "w-huber": (True, "huber"), "huber": (False, "huber")}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", list(CASES))
def test_f64_update_w_vs_autograd_and_oracle(dqn_golden, case, variant, loss_kind_reset):
    """3 updates of B = 256 (the hard update after the third): float64 loss and every gradient entry within 1e-12 relative of
    torch autograd (entries that cancel to near 0: 1e-15 of the largest); against the oracle (fp32 networks, double accumulation) loss within 2e-5 relative, gradient within 2e-4,
    |q_a - y| within abs_err_bound.  Both losses' branches and zero / one weights are exercised."""
    in_dim, hidden, n_actions, dueling, algo = CASES[case]
    weighted, kind = VARIANTS[variant]
    B = 256
    rng = np.random.default_rng(sum(map(ord, case + variant)))
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    net = O.make_net(in_dim, hidden, n_actions, dueling)
    P = sum(o * i + o for o, i in layers)
    assert P == O.net_param_count(net)
    local0 = rng.normal(0, 0.15, P).astype(np.float32)
    OL = O.OracleLearner(net, algo, local0, update_loop=3)
    OL.target[:] = rng.normal(0, 0.15, P).astype(np.float32)
    O.set_loss_kind(kind)
    for step in range(3):
        s, a, r, s2, d, w, redrawn = draw_batch(dqn_golden, rng, layers, dueling, algo, [OL.local], OL.target, B, in_dim,
                                                n_actions, kind, weighted)
        assert max(redrawn.values()) <= 0.05 * B, redrawn
        l64, g64, ae64, y64 = f64_update(layers, algo, dueling, OL.local, OL.target, s, a, r, s2, d, w, kind)
        lt, gt = torch_update(layers, algo, dueling, OL.local, OL.target, s, a, r, s2, d, w, kind)
        assert abs(l64 - lt) <= 1e-12 * abs(lt), (step, l64, lt)
        # relative per entry; an entry that cancels to near 0 keeps a floor of 1e-15 of the largest (a few float64 ulps of
        # the terms it summed)
        assert (np.abs(g64 - gt) <= 1e-12 * (np.abs(gt) + 1e-3 * np.abs(gt).max())).all(), (step, float(np.abs(g64 - gt).max()))
        if kind == "huber":
            assert (ae64 < 1).mean() >= 0.1 and (ae64 > 1).mean() >= 0.1, (ae64 < 1).mean()
        if weighted:
            assert (w == 0).any() and (w == 1).any() and ((w > 0) & (w < 1)).any()
        lo, go, aeo = OL.update(s, a, r, s2, d, is_w=np.ones(B, np.float32) if w is None else w)
        assert np.isclose(lo, l64, rtol=2e-5, atol=0), (step, lo, l64)
        assert np.abs(go - g64).max() <= 2e-4, (step, float(np.abs(go - g64).max()))
        err = np.abs(aeo - ae64) - abs_err_bound(y64, r, ae64)
        assert (err <= 0).all(), (step, float(err.max()))
