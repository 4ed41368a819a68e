"""The float64 restatement of the Q-network forward pass and of one TD update, with the batch draws the sweeps feed the
kernels.  It is the one arbiter between fp32 implementations whose summation orders differ, and it is pinned to torch
autograd and to the CPU oracle in test_weighted_f64_cpu.py before any GPU test compares against it.  Also the judges of sampled
updates and actions the loops' tests share: the entries a row near a ReLU kink may move, the double-DQN tie allowance, the
tally that keeps both rare, and the eps-greedy / argmax check of an act call."""
import numpy as np
import pytest

import oracle as O
import replay_restatement as R

GAMMA = 0.99


def net_layers(in_dim, hidden, n_actions, dueling):
    """(out, in) of every Linear in state_dict order: the trunk, then fc_A (or the Q head) and fc_V."""
    dims = [in_dim] + list(hidden)
    head = [(n_actions, hidden[-1]), (1, hidden[-1])] if dueling else [(n_actions, hidden[-1])]
    return [(dims[i + 1], dims[i]) for i in range(len(hidden))] + head


def f64_unpack(layers, flat):
    out, off = [], 0
    for (o, i) in layers:
        W = flat[off:off + o * i].reshape(o, i).astype(np.float64); off += o * i
        b = flat[off:off + o].astype(np.float64); off += o
        out.append((W, b))
    assert off == flat.size
    return out


def f64_forward(P, dueling, x):
    """Q(x) of the unpacked float64 network P, and the activations [x, H1, ..] kept for the backward pass."""
    x = np.asarray(x, np.float64)
    acts, h = [x], x
    nt = len(P) - (2 if dueling else 1)
    for W, b in P[:nt]:
        h = np.maximum(h @ W.T + b, 0.0); acts.append(h)
    if dueling:
        (WA, bA), (WV, bV) = P[nt], P[nt + 1]
        A = h @ WA.T + bA; V = h @ WV.T + bV
        return V + A - A.mean(1, keepdims=True), acts
    W, b = P[nt]
    return h @ W.T + b, acts


def big_inputs(g, n, rng, in_dim=100):
    """n rows of the golden observations (columns cropped or tiled to in_dim) plus noise: occupancy bits and real-valued
    entries at the scales the learner sees."""
    base = np.concatenate([g["batch_s"].reshape(-1, 100), g["batch_s2"].reshape(-1, 100)])
    base = np.tile(base, (1, -(-in_dim // 100)))[:, :in_dim]
    x = np.tile(base, (n // base.shape[0] + 1, 1))[:n]
    return (x + rng.normal(0, 0.02, x.shape)).astype(np.float32)


def near_relu_kink(P, dueling, x, rel=2e-5):
    """Rows of x for which a hidden pre-activation of the float64 network P lies within rel x (the sum of its terms'
    magnitudes) of 0: 3xTF32 products (2^-21) and fp32 sums over <= 128 terms stay well inside that."""
    h = np.asarray(x, np.float64)
    near = np.zeros(h.shape[0], bool)
    for W, b in P[:len(P) - (2 if dueling else 1)]:
        z = h @ W.T + b
        near |= (np.abs(z) <= rel * (np.abs(h) @ np.abs(W).T + np.abs(b))).any(1)
        h = np.maximum(z, 0.0)
    return near


def f64_update(layers, algo, dueling, local, target, s, a, r, s2, d, w=None, loss_kind="mse", gamma=GAMMA, abs_terms=False):
    """One TD update in float64 numpy with per-sample importance weights w (None = all 1) -> (loss, gradient in state_dict
    order, |q_a - y| per sample, y).  The forms the kernels document (learner.cu update_kernel, tc_train.cu head epilogue):
    MSE: loss = mean(w diff^2), dL/dq_a = 2 w diff / B;  Huber (SmoothL1, beta = 1): loss = mean(w h(diff)) with
    h = 0.5 diff^2 below |diff| = 1 and |diff| - 0.5 above, dL/dq_a = w clip(diff, -1, 1) / B.  diff = q_a - y, y = r + gamma
    max_a' q_target(s') (DQN) or q_target(s', argmax q_local(s')) (DDQN / dueling), times (1 - d).  These are
    DQN_Trainer.py:107-124 / DDQN_Trainer.py:93-107 / DuelingDQN_Trainer.py:164-180 with the weights and the loss kind added.
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
    _, _, _, y0 = f64_update(layers, algo, dueling, local, target, s, a, zero, s2, d)
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


# ------------------------------------------------------------------ judging sampled updates and actions
def trunk_exempt(layers, n_trunk, P64, dueling, s, rel=2e-5):
    """Gradient entries the rows of s near a ReLU kink can move: for a unit of trunk layer l near its kink on some row, that
    unit's weight row and bias and every entry of the layers below l.  Returns (mask, number of kink rows)."""
    offs, o = [], 0
    for (n_out, n_in) in layers:
        offs.append((o, o + n_out * n_in, n_out, n_in)); o += n_out * n_in + n_out
    mask = np.zeros(o, bool)
    h = np.asarray(s, np.float64)
    rows = np.zeros(h.shape[0], bool)
    for l, (W, b) in enumerate(P64[:n_trunk]):
        z = h @ W.T + b
        near = np.abs(z) <= rel * (np.abs(h) @ np.abs(W).T + np.abs(b))
        units = np.flatnonzero(near.any(0))
        rows |= near.any(1)
        w0, b0, n_out, n_in = offs[l]
        for j in units:
            mask[w0 + j * n_in:w0 + (j + 1) * n_in] = True
            mask[b0 + j] = True
        if units.size:
            mask[:offs[l][0]] = True
        h = np.maximum(z, 0.0)
    return mask, int(rows.sum())


def tie_allowance(layers, algo, dueling, local, target, batch, P, gamma=GAMMA):
    """Double-DQN rows whose next-state top-2 local values tie within 1e-4: the loss and gradient change that choosing the
    other action would make (row b moves y by delta_b = gamma |q_T(s2, a1) - q_T(s2, a2)| (1 - d); the gradient by
    (2 / B) delta_b |dQ(s_b, a_b) / dtheta|).  Returns (loss allowance, gradient allowance [P], tied rows)."""
    s, a, r, s2, d = batch
    B = s.shape[0]
    gal = np.zeros(P)
    if algo == O.ALGO_DQN:
        return 0.0, gal, 0
    PL, PT = f64_unpack(layers, local), f64_unpack(layers, target)
    ql = f64_forward(PL, dueling, s2)[0]
    order = np.argsort(ql, 1)
    top, second = order[:, -1], order[:, -2]
    tie = (ql[np.arange(B), top] - ql[np.arange(B), second] < 1e-4) & (d == 0)
    rows = np.flatnonzero(tie)
    if not rows.size:
        return 0.0, gal, 0
    qt = f64_forward(PT, dueling, s2[rows])[0]
    delta = gamma * np.abs(qt[np.arange(rows.size), top[rows]] - qt[np.arange(rows.size), second[rows]])
    q = f64_forward(PL, dueling, s[rows])[0][np.arange(rows.size), a[rows]]
    y = r[rows] + gamma * qt[np.arange(rows.size), top[rows]]
    lal = float(np.sum(delta * (2 * np.abs(q - y) + delta)) / B)
    for k, b in enumerate(rows):
        one = lambda rr: f64_update(layers, algo, dueling, local, target, s[b:b + 1], a[b:b + 1], np.array([rr], np.float32),  # noqa: E731
                                    s2[b:b + 1], np.zeros(1, np.float32), gamma=gamma)[1]
        J = (one(0.0) - one(1.0)) / 2.0                        # dQ(s_b, a_b) / dtheta
        gal += (2.0 / B) * delta[k] * np.abs(J)
    return lal, gal * 1.01, int(rows.size)


class Tally:
    """Counts of the sampled rows near a kink or a tie over a leg: they must stay rare.  (One such row in a deep layer moves
    every entry of the layers below it, so the exempted entries are counted but not bounded.)"""

    def __init__(self):
        self.rows = self.kink_rows = self.tie_rows = self.entries = self.exempt = 0

    def check(self):
        assert self.rows > 0
        assert self.kink_rows <= 0.05 * self.rows + 2, (self.kink_rows, self.rows)
        assert self.tie_rows <= 0.02 * self.rows + 2, (self.tie_rows, self.rows)


def check_actions(s, a, seed, call, p_before, eps, shape, G=1):
    """Actions a of the rows s that act call `call` of a learner seeded with `seed` chose (G equal trainer blocks): the restated
    eps-greedy draw on random rows, the float64 argmax of the parameters before the call (p_before[g]) on greedy rows where the
    top-2 gap exceeds 1e-4."""
    in_dim, hidden, n_actions, dueling = shape
    layers = net_layers(in_dim, hidden, n_actions, dueling)
    N = s.shape[0]
    Ng = N // G
    n_clear = 0
    for g in range(G):
        rows = slice(g * Ng, (g + 1) * Ng)
        greedy, ra = R.eps_greedy(seed, call, Ng, eps, n_actions, g)
        ag = a[rows]
        assert np.array_equal(ag[~greedy], ra[~greedy]), (g, call)
        q = f64_forward(f64_unpack(layers, p_before[g]), dueling, s[rows])[0]
        top2 = np.sort(q, 1)[:, -2:]
        clear = greedy & ((top2[:, 1] - top2[:, 0]) > 1e-4)
        assert np.array_equal(ag[clear], q[clear].argmax(1)), (g, call, int((ag[clear] != q[clear].argmax(1)).sum()))
        n_clear += int(clear.sum()) + int((~greedy).sum())
    assert n_clear >= 0.98 * N


@pytest.fixture
def loss_kind_reset():
    yield
    O.set_loss_kind("mse")            # the oracle's loss kind is process-wide state
