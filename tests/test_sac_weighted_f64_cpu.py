"""The weighted (prioritised-replay) form of the float64 SAC restatement, sac_update64_weighted, pinned before it judges the
weighted critic kernel: w = 1 is the uniform update, and random weights agree with an independent torch float64 autograd
statement of the networks and the weighted losses (include/uavrl.h, the prioritised-replay block).  No GPU."""
import numpy as np
import torch

from sac_restatement import HP, draw_batch, init_state, sac_update64
from sac_weighted_restatement import sac_update64_weighted

A = 2


def _nets(p, kind, obs, hid):
    """Flat state_dict-ordered vector -> torch float64 leaf tensors (W, b) per layer."""
    shapes = [(hid, obs), (A, hid), (A, hid)] if kind == "actor" else [(hid, obs + A), (hid, hid), (A, hid)]
    out, o = [], 0
    for n_out, n_in in shapes:
        W = torch.tensor(p[o:o + n_out * n_in].reshape(n_out, n_in), dtype=torch.float64, requires_grad=True); o += n_out * n_in
        b = torch.tensor(p[o:o + n_out], dtype=torch.float64, requires_grad=True); o += n_out
        out.append((W, b))
    return out


def _actor(P, s, eps, bound):
    (W1, b1), (Wm, bm), (Ws, bs) = P
    h = torch.relu(s @ W1.T + b1)
    mu, sd = torch.tanh(h @ Wm.T + bm), torch.tanh(torch.nn.functional.softplus(h @ Ws.T + bs))
    xs = mu + sd * eps
    lp = torch.distributions.Normal(mu, sd).log_prob(xs)
    a = torch.tanh(xs)
    return a * bound, lp - torch.log(1 - torch.tanh(a) ** 2 + 1e-7)


def _critic(P, s, a):
    (W1, b1), (W2, b2), (W3, b3) = P
    h = torch.relu(torch.cat([s, a], 1) @ W1.T + b1)
    return torch.relu(h @ W2.T + b2) @ W3.T + b3


def _adam(p, m, v, g, lr, t):
    m = 0.9 * m + 0.1 * g
    v = 0.999 * v + 0.001 * g * g
    return p - lr / (1 - 0.9 ** t) * m / (np.sqrt(v) / np.sqrt(1 - 0.999 ** t) + 1e-8), m, v


def _flat_grad(P):
    return np.concatenate([np.concatenate([W.grad.numpy().ravel(), b.grad.numpy()]) for W, b in P])


def _flat(P):
    return np.concatenate([np.concatenate([W.detach().numpy().ravel(), b.detach().numpy()]) for W, b in P])


def torch_weighted_update(st, s, a, r, s2, d, e1, e2, w, obs, hid, bound, hp=HP):
    """SAC_Trainer.update (continuous) with the port's weighted critic losses, by torch autograd in float64."""
    T = lambda x: torch.tensor(np.asarray(x, np.float64))                    # noqa: E731
    s, a, r, s2, d, e1, e2, w = map(T, (s, a, r, s2, d, e1, e2, w))
    t = st["step"] + 1
    new = dict(st, step=t)
    log_alpha = torch.tensor(st["log_alpha"], dtype=torch.float64, requires_grad=True)
    alpha = log_alpha.exp().detach()
    actor = _nets(st["actor"], "actor", obs, hid)
    c = [_nets(st[k], "critic", obs, hid) for k in ("c1", "c2")]
    tc = [_nets(st[k], "critic", obs, hid) for k in ("t1", "t2")]
    with torch.no_grad():
        an, lpn = _actor(actor, s2, e1, bound)
        y = r[:, None] + hp["gamma"] * (torch.minimum(_critic(tc[0], s2, an), _critic(tc[1], s2, an)) - alpha * lpn) * (1 - d[:, None])
    q = [_critic(c[i], s, a) for i in (0, 1)]
    e_b = (torch.minimum(q[0], q[1]) - y).abs().mean(1).detach().numpy()
    out = {"abs_err": e_b}
    for i, k in enumerate(("c1", "c2")):
        loss = (w[:, None] * (q[i] - y) ** 2).mean()
        loss.backward()
        out["l_" + k] = loss.item()
        new[k], new[k + "_m"], new[k + "_v"] = _adam(st[k], st[k + "_m"], st[k + "_v"], _flat_grad(c[i]), hp["critic_lr"], t)
    cn = [_nets(new[k], "critic", obs, hid) for k in ("c1", "c2")]
    act, lp = _actor(actor, s, e2, bound)
    la = (alpha * lp - torch.minimum(_critic(cn[0], s, act), _critic(cn[1], s, act))).mean()
    la.backward()
    out["l_actor"] = la.item()
    new["actor"], new["actor_m"], new["actor_v"] = _adam(st["actor"], st["actor_m"], st["actor_v"], _flat_grad(actor), hp["actor_lr"], t)
    ent = (-lp).mean().detach()
    alpha_loss = ((ent - hp["target_entropy"]) * log_alpha.exp()).mean()
    alpha_loss.backward()
    out["g_alpha"] = log_alpha.grad.item()
    new["log_alpha"], new["la_m"], new["la_v"] = _adam(st["log_alpha"], st["la_m"], st["la_v"], out["g_alpha"], hp["alpha_lr"], t)
    for k in ("1", "2"):
        new["t" + k] = st["t" + k] * (1 - hp["tau"]) + new["c" + k] * hp["tau"]
    return new, out


KEYS = ("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v", "log_alpha", "la_m", "la_v")


def test_unit_weights_are_the_uniform_update():
    """w = 1 gives sac_update64's uniform update to float64 rounding: every parameter, moment, alpha word, loss, reduced
    gradient and its bound, loss scale and network evaluation the GPU checks read."""
    rng = np.random.default_rng(5)
    for obs, hid, bound, B in ((100, 64, 1.0, 64), (12, 17, 0.5, 45)):
        st = init_state(rng, obs, hid)
        batch = draw_batch(rng, B, obs, bound)
        new0, out0 = sac_update64(st, *batch, obs, hid, bound)
        new1, out1 = sac_update64_weighted(st, *batch, obs, hid, bound, np.ones(B))
        for k in KEYS:
            np.testing.assert_allclose(new1[k], new0[k], rtol=1e-13, atol=1e-15, err_msg=k)
        np.testing.assert_allclose(out1["losses"], out0["losses"], rtol=1e-13, atol=1e-15)
        for k in ("actor", "c1", "c2"):
            for part in ("grads", "gabs"):
                np.testing.assert_allclose(out1[part][k], out0[part][k], rtol=1e-12, atol=1e-15, err_msg=part + " " + k)
        for k in ("lscale_c1", "lscale_c2", "lscale_actor", "ascale"):
            np.testing.assert_allclose(out1[k], out0[k], rtol=1e-13, err_msg=k)
        for e1, e0 in zip(out1["evals"], out0["evals"]):
            for k in e0:
                np.testing.assert_allclose(e1[k], e0[k], rtol=1e-13, atol=1e-15, err_msg=k)
        assert "abs_err" not in out0 and out1["abs_err"].shape == (B,)


def test_random_weights_agree_with_torch_autograd():
    """Random importance weights, exact 0 and 1 among them, over three chained updates at two shapes: sac_update64_weighted and
    the torch float64 autograd statement agree on parameters, moments, log_alpha, the three losses and e_b."""
    rng = np.random.default_rng(9)
    for obs, hid, bound, B in ((100, 64, 1.0, 64), (12, 17, 0.5, 37)):
        st = init_state(rng, obs, hid)
        for _ in range(3):
            batch = draw_batch(rng, B, obs, bound)
            w = rng.uniform(0, 1, B)
            w[:3] = 0.0
            w[3:6] = 1.0
            new, out = sac_update64_weighted(st, *batch, obs, hid, bound, w)
            ref, rout = torch_weighted_update(st, *batch, w, obs, hid, bound)
            for k in KEYS:
                np.testing.assert_allclose(new[k], ref[k], rtol=1e-9, atol=1e-12, err_msg=k)
            np.testing.assert_allclose([out["l_actor"], out["l_c1"], out["l_c2"]], [rout["l_actor"], rout["l_c1"], rout["l_c2"]],
                                       rtol=1e-10)
            np.testing.assert_allclose(out["abs_err"], rout["abs_err"], rtol=1e-12, atol=1e-14)
            st = new
