"""The float64 restatement of the prioritised-replay / Huber update (f64_update_w), pinned before it judges any kernel: against
torch autograd on the same float64 network (to 1e-12) and against the CPU oracle's weighted update (ora_dqn_update_per under
both loss kinds, at the fp32 bounds test_tc_update_large_batch_vs_oracle uses).  draw_batch builds the batches the GPU sweep
(test_weighted_update_shapes_gpu.py) feeds the kernels, with the samples whose float64 value sits on a discontinuity redrawn."""
import numpy as np
import pytest
import torch

import oracle as O
from test_qnet_shapes_gpu import near_relu_kink
from test_tc_gpu import big_inputs, f64_forward, f64_unpack, net_layers

GAMMA = 0.99


def f64_update_w(layers, algo, dueling, local, target, s, a, r, s2, d, w=None, loss_kind="mse", gamma=GAMMA, abs_terms=False):
    """One TD update in float64 numpy with per-sample importance weights w (None = all 1) -> (loss, gradient in state_dict
    order, |q_a - y| per sample, y).  The forms the kernels document (learner.cu update_kernel, tc_train.cu head epilogue):
    MSE: loss = mean(w diff^2), dL/dq_a = 2 w diff / B;  Huber (SmoothL1, beta = 1): loss = mean(w h(diff)) with
    h = 0.5 diff^2 below |diff| = 1 and |diff| - 0.5 above, dL/dq_a = w clip(diff, -1, 1) / B.  diff = q_a - y, y = r + gamma
    max_a' q_target(s') (DQN) or q_target(s', argmax q_local(s')) (DDQN / dueling), times (1 - d).
    abs_terms: also return, per gradient entry, the sum over samples of the magnitudes of the products it adds up (the scale
    of an fp32-grade implementation's rounding error in that entry)."""
    PL, PT = f64_unpack(layers, local), f64_unpack(layers, target)
    B = s.shape[0]
    rows = np.arange(B)
    qt, _ = f64_forward(PT, dueling, s2)
    nq = qt.max(1) if algo == 0 else qt[rows, f64_forward(PL, dueling, s2)[0].argmax(1)]
    y = r.astype(np.float64) + gamma * nq * (1.0 - d.astype(np.float64))
    q, acts = f64_forward(PL, dueling, s)
    diff = q[rows, a] - y
    wb = np.ones(B) if w is None else w.astype(np.float64)
    ad = np.abs(diff)
    if loss_kind == "mse":
        loss = float((wb * diff ** 2).mean())
        dq = 2.0 * wb * diff / B
    else:
        loss = float((wb * np.where(ad < 1.0, 0.5 * diff ** 2, ad - 0.5)).mean())
        dq = wb * np.clip(diff, -1.0, 1.0) / B
    gq = np.zeros_like(q); gq[rows, a] = dq
    nt = len(PL) - (2 if dueling else 1)
    h = acts[-1]
    if dueling:
        gA = gq - gq.sum(1, keepdims=True) / q.shape[1]; gV = gq.sum(1, keepdims=True)
        gh = gA @ PL[nt][0] + gV @ PL[nt + 1][0]
        heads = [(gA, h), (gV, h)]
    else:
        gh = gq @ PL[nt][0]
        heads = [(gq, h)]
    terms = []
    for l in range(nt - 1, -1, -1):
        gz = gh * (acts[l + 1] > 0)
        terms = [(gz, acts[l])] + terms
        gh = gz @ PL[l][0]
    terms += heads
    grad = np.concatenate([x for gz, x in terms for x in ((gz.T @ x).ravel(), gz.sum(0))])
    if not abs_terms:
        return loss, grad, ad, y
    mag = np.concatenate([m for gz, x in terms for m in ((np.abs(gz).T @ np.abs(x)).ravel(), np.abs(gz).sum(0))])
    return loss, grad, ad, y, mag


def abs_err_bound(y, r, ae):
    """How far an fp32-grade |q_a - y| may lie from float64: q of the act tests' bound (2e-5 + 2e-5 |q|) on q_a and, through
    gamma, on the next-state value nq, plus one fp32 rounding in each of gamma nq, r + gamma nq and q_a - y.  With
    |q_a| <= |y| + |diff| and gamma |nq| <= |y| + |r| this is 2e-5 (1 + gamma) + 2e-5 (2 |y| + |r| + |diff|) +
    2^-23 (|y| + |r| + |diff|)."""
    y, r, ae = np.abs(y), np.abs(np.asarray(r, np.float64)), np.abs(ae)
    return 2e-5 * (1.0 + GAMMA) + 2e-5 * (2.0 * y + r + ae) + 2.0 ** -23 * (y + r + ae)


def draw_batch(g, rng, layers, dueling, algo, locals_, target, B, in_dim, n_actions, loss_kind, weighted):
    """A batch of B transitions for the networks (locals_: the local parameter vectors every implementation under test
    holds, target: the target parameters) -> (s, a, r, s2, d, w, redrawn), where redrawn counts the samples moved off a
    discontinuity of the float64 function:
      - 'kink': a hidden pre-activation of s within fp32 noise of 0 (near_relu_kink): s is drawn again;
      - 'tie': DDQN / dueling next-state action whose two best local values lie within 1e-3: marked terminal;
      - 'branch': Huber |diff64| within 1e-3 of 1, where the two branches meet: its TD error is drawn again.
    MSE batches draw r ~ N(0, 1) as the shape sweep does; Huber batches set the rewards so that diff64 = q_a - y ~ N(0, 1.5),
    about half of the samples on each branch (the clipped gradient does not grow with diff).  Weights (when weighted) are
    uniform in (0, 1] with about 10 % exact 1 and 5 % exact 0."""
    redrawn = dict(kink=0, tie=0, branch=0)
    Ps = [f64_unpack(layers, p) for p in locals_]
    s = big_inputs(g, B, rng, in_dim); s2 = big_inputs(g, B, rng, in_dim)
    for it in range(20):
        kink = np.zeros(B, bool)
        for P in Ps:
            kink |= near_relu_kink(P, dueling, s)
        if not kink.any():
            break
        if it == 0:
            redrawn["kink"] = int(kink.sum())
        s[kink] = big_inputs(g, int(kink.sum()), rng, in_dim)
    assert not kink.any()
    a = rng.integers(0, n_actions, B).astype(np.int32)
    d = (rng.uniform(size=B) < 0.1).astype(np.float32)
    if algo != 0:
        tie = np.zeros(B, bool)
        for P in Ps:
            ql = np.sort(f64_forward(P, dueling, s2)[0], 1)
            tie |= (ql[:, -1] - ql[:, -2]) < 1e-3
        redrawn["tie"] = int((tie & (d == 0)).sum())
        d[tie] = 1.0
    if loss_kind != "huber":
        r = rng.normal(0.0, 1.0, B).astype(np.float32)
    else:
        r = huber_rewards(rng, layers, dueling, algo, Ps, locals_[0], target, s, a, s2, d, redrawn)
    w = None
    if weighted:
        w = (1.0 - rng.random(B)).astype(np.float32)
        u = rng.random(B)
        w[u < 0.1] = 1.0
        w[u > 0.95] = 0.0
    return s, a, r, s2, d, w, redrawn


def huber_rewards(rng, layers, dueling, algo, Ps, local, target, s, a, s2, d, redrawn):
    """Rewards with diff64 ~ N(0, 1.5) and no |diff64| within 1e-3 of the branch point under any of the local networks Ps."""
    B = s.shape[0]
    zero = np.zeros(B, np.float32)
    qa = [f64_forward(P, dueling, s)[0][np.arange(B), a] for P in Ps]
    _, _, _, y0 = f64_update_w(layers, algo, dueling, local, target, s, a, zero, s2, d)
    t = rng.normal(0.0, 1.5, B)
    for it in range(20):
        r = (qa[0] - y0 - t).astype(np.float32)
        near = np.zeros(B, bool)
        for q in qa:
            near |= np.abs(np.abs(q - y0 - r) - 1.0) < 1e-3
        if not near.any():
            break
        if it == 0:
            redrawn["branch"] = int(near.sum())
        t[near] = rng.normal(0.0, 1.5, int(near.sum()))
    assert not near.any()
    return r


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


@pytest.fixture
def loss_kind_reset():
    yield
    O.set_loss_kind("mse")            # the oracle's loss kind is process-wide state


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
        l64, g64, ae64, y64 = f64_update_w(layers, algo, dueling, OL.local, OL.target, s, a, r, s2, d, w, kind)
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
