"""The float64 restatement of one SAC_Trainer.update (continuous; Trainer/SAC_Trainer.py:122-147, 325-379;
BaseClass/BaseCNN.py:459-500), the batch draws the SAC sweeps feed the learner, and check_step, which holds one learner step
to the float64 one.  It is pinned to the reference's own run (tests/golden/sac_golden.npz) and to the CPU oracle in
test_sac_f64_cpu.py before any GPU test compares against it."""
import numpy as np

A = 2                                       # action_dim of the UAV task
HP = dict(actor_lr=1e-4, critic_lr=1e-3, alpha_lr=1e-4, target_entropy=1.0, gamma=0.99, tau=0.05)


def unpack(p, kind, obs, hid):
    """Flat state_dict-ordered vector -> list of (W [out][in], b [out]): actor fc1, fc_mu, fc_std; critic fc1, fc2, fc_out."""
    p = np.asarray(p, np.float64)
    shapes = [(hid, obs), (A, hid), (A, hid)] if kind == "actor" else [(hid, obs + A), (hid, hid), (A, hid)]
    out, o = [], 0
    for n_out, n_in in shapes:
        W = p[o:o + n_out * n_in].reshape(n_out, n_in); o += n_out * n_in
        b = p[o:o + n_out]; o += n_out
        out.append((W, b))
    assert o == p.size
    return out


def flat(grads):
    return np.concatenate([np.concatenate([gW.ravel(), gb]) for gW, gb in grads])


def softplus(x):
    return np.where(x > 20.0, x, np.log1p(np.exp(np.minimum(x, 20.0))))      # F.softplus, threshold 20


def actor_fwd(P, s, eps, bound):
    """PolicyNetContinuous_SAC.forward (BaseCNN.py:471-483): rsample, tanh squash, the log-prob correction with tanh applied
    twice (:481).  Returns the cache the backward needs; 'act' = action * bound."""
    (W1, b1), (Wm, bm), (Ws, bs) = P
    z = s @ W1.T + b1
    h = np.maximum(z, 0.0)
    pm, ps = h @ Wm.T + bm, h @ Ws.T + bs
    mu, sd = np.tanh(pm), np.tanh(softplus(ps))
    xs = mu + sd * eps
    lp = -((xs - mu) ** 2) / (2.0 * sd * sd) - np.log(sd) - 0.5 * np.log(2.0 * np.pi)
    a = np.tanh(xs)
    t = np.tanh(a)
    logp = lp - np.log(1.0 - t * t + 1e-7)
    zabs = np.abs(s) @ np.abs(W1).T + np.abs(b1)
    return dict(s=s, z=z, zabs=zabs, h=h, hm=mag(h, z, zabs), pm=pm, ps=ps, mu=mu, sd=sd, a=a, t=t, logp=logp, act=a * bound, eps=eps)


def mag(h, z, zabs):
    """Magnitude of a ReLU activation for the gradient bounds: its value plus 1 % of the sum of its terms' magnitudes (an
    activation just above 0 carries the fp32 error of that sum, not of its small value)."""
    return h + 0.01 * zabs * (z > 0)


def critic_fwd(P, s, act):
    (W1, b1), (W2, b2), (W3, b3) = P
    x = np.concatenate([s, act], 1)
    z1 = x @ W1.T + b1; h1 = np.maximum(z1, 0.0)
    z2 = h1 @ W2.T + b2; h2 = np.maximum(z2, 0.0)
    q = h2 @ W3.T + b3
    z1abs, z2abs = np.abs(x) @ np.abs(W1).T + np.abs(b1), h1 @ np.abs(W2).T + np.abs(b2)
    return dict(x=x, z1=z1, h1=h1, z2=z2, h2=h2, q=q, z1abs=z1abs, z2abs=z2abs, qabs=h2 @ np.abs(W3).T + np.abs(b3),
                h1m=mag(h1, z1, z1abs), h2m=mag(h2, z2, z2abs))


def critic_bwd(P, c, dq, dq_mag):
    """dq [B, A] -> (parameter gradients, their magnitude bounds, d/d action input [B, A], its magnitude bound).  The bounds run
    the same chain on magnitudes (dq_mag, |W|): what every sum in the chain adds up before it cancels, which is what an
    fp32 evaluation's error scales with."""
    (W1, _), (W2, _), (W3, _) = P
    dz2 = (dq @ W3) * (c["z2"] > 0); m2 = (dq_mag @ np.abs(W3)) * (c["z2"] > 0)
    dz1 = (dz2 @ W2) * (c["z1"] > 0); m1 = (m2 @ np.abs(W2)) * (c["z1"] > 0)
    g = [(dz1.T @ c["x"], dz1.sum(0)), (dz2.T @ c["h1"], dz2.sum(0)), (dq.T @ c["h2"], dq.sum(0))]
    ga = [(m1.T @ np.abs(c["x"]), m1.sum(0)), (m2.T @ c["h1m"], m2.sum(0)), (dq_mag.T @ c["h2m"], dq_mag.sum(0))]
    obs = c["x"].shape[1] - A
    return g, ga, (dz1 @ W1)[:, obs:], (m1 @ np.abs(W1))[:, obs:]


def adam(p, m, v, g, lr, t):
    """torch.optim.Adam's single-tensor step in the form reduce_adam_kernel computes it (lerp, mul/addcmul, sqrt / sqrt(bc2)
    + eps, addcdiv with lr / bc1)."""
    bc1, bc2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
    m = m + (g - m) * 0.1
    v = v * 0.999 + 0.001 * g * g
    return p - (lr / bc1) * (m / (np.sqrt(v) / np.sqrt(bc2) + 1e-8)), m, v


def sac_update64(st, s, a, r, s2, d, eps_next, eps_cur, obs, hid, bound, hp=HP):
    """One SAC_Trainer.update (continuous) in float64 from state st (dict: actor, c1, c2, t1, t2, their Adam moments
    actor_m.. c2_v, log_alpha, la_m, la_v, step).  Returns (new state, out) where out holds the four loss outputs, the three
    reduced gradients, their magnitude bounds (critic_bwd), and what the noise checks need."""
    f = lambda x: np.asarray(x, np.float64)                                            # noqa: E731
    s, a, r, s2, d, eps_next, eps_cur = map(f, (s, a, r, s2, d, eps_next, eps_cur))
    B = s.shape[0]
    nel = float(B * A)
    alpha = np.exp(st["log_alpha"])
    t = st["step"] + 1
    new = dict(st, step=t)
    Pa = unpack(st["actor"], "actor", obs, hid)
    Pc = [unpack(st[k], "critic", obs, hid) for k in ("c1", "c2", "t1", "t2")]
    # calc_target (:122-131): [B, A]-shaped
    an = actor_fwd(Pa, s2, eps_next, bound)
    ct = [critic_fwd(Pc[2], s2, an["act"]), critic_fwd(Pc[3], s2, an["act"])]
    td = r[:, None] + hp["gamma"] * (np.minimum(ct[0]["q"], ct[1]["q"]) - alpha * an["logp"]) * (1.0 - d[:, None])
    tdabs = np.abs(r)[:, None] + hp["gamma"] * (np.maximum(ct[0]["qabs"], ct[1]["qabs"]) + alpha * np.abs(an["logp"]))
    out = dict(evals=[an, ct[0], ct[1]], grads={}, gabs={})
    # critics (:343-360)
    for i, k in enumerate(("c1", "c2")):
        c = critic_fwd(Pc[i], s, a)
        diff = c["q"] - td
        out["l_" + k] = np.mean(diff * diff)
        out["lscale_" + k] = np.mean(np.abs(diff) * (np.abs(c["q"]) + np.abs(td) + 1.0))
        # Q - y may cancel: its error scales with |Q| + |y|, so the magnitude carries 1 % of that
        g, ga, _, _ = critic_bwd(Pc[i], c, 2.0 * diff / nel, 2.0 * (np.abs(diff) + 0.01 * (c["qabs"] + tdabs)) / nel)
        out["grads"][k], out["gabs"][k] = flat(g), flat(ga)
        new[k], new[k + "_m"], new[k + "_v"] = adam(st[k], st[k + "_m"], st[k + "_v"], out["grads"][k], hp["critic_lr"], t)
        out["evals"].append(c)
    # actor (:362-369) with the updated critics
    Pn = [unpack(new[k], "critic", obs, hid) for k in ("c1", "c2")]
    ac = actor_fwd(Pa, s, eps_cur, bound)
    q = [critic_fwd(Pn[0], s, ac["act"]), critic_fwd(Pn[1], s, ac["act"])]
    q1, q2 = q[0]["q"], q[1]["q"]
    out["l_actor"] = np.mean(alpha * ac["logp"] - np.minimum(q1, q2))
    out["lscale_actor"] = np.mean(np.abs(alpha * ac["logp"]) + np.abs(np.minimum(q1, q2)))
    gmin = -1.0 / nel                                                                  # d loss / d min(q1, q2): torch splits ties
    dq1 = np.where(q1 < q2, gmin, np.where(q1 > q2, 0.0, 0.5 * gmin))
    dq2 = np.where(q2 < q1, gmin, np.where(q2 > q1, 0.0, 0.5 * gmin))
    _, _, da1, da1m = critic_bwd(Pn[0], q[0], dq1, np.abs(dq1))
    _, _, da2, da2m = critic_bwd(Pn[1], q[1], dq2, np.abs(dq2))
    glogp = alpha / nel
    tt, aa = ac["t"], ac["a"]
    dc_da = 2.0 * tt * (1.0 - tt * tt) / (1.0 - tt * tt + 1e-7)                          # d -log(1 - tanh(a)^2 + 1e-7) / da
    dxs = (da1 + da2) * bound * (1.0 - aa * aa) + glogp * dc_da * (1.0 - aa * aa)
    dsd = dxs * ac["eps"] + glogp * (-1.0 / ac["sd"])                                   # d log N(xs; mu, sd) / d sd = -1 / sd
    dpm = dxs * (1.0 - ac["mu"] ** 2)
    sig = np.where(ac["ps"] > 20.0, 1.0, 1.0 / (1.0 + np.exp(-ac["ps"])))                  # d softplus / d ps
    dps = dsd * (1.0 - ac["sd"] ** 2) * sig
    xm = (da1m + da2m) * bound * (1.0 - aa * aa) + glogp * np.abs(dc_da) * (1.0 - aa * aa)      # magnitude chain, as critic_bwd
    pmm, psm = xm * (1.0 - ac["mu"] ** 2), (xm * np.abs(ac["eps"]) + glogp / ac["sd"]) * (1.0 - ac["sd"] ** 2) * sig
    (W1, _), (Wm, _), (Ws, _) = Pa
    dz = (dpm @ Wm + dps @ Ws) * (ac["z"] > 0)
    zm = (pmm @ np.abs(Wm) + psm @ np.abs(Ws)) * (ac["z"] > 0)
    g = [(dz.T @ s, dz.sum(0)), (dpm.T @ ac["h"], dpm.sum(0)), (dps.T @ ac["h"], dps.sum(0))]
    ga = [(zm.T @ np.abs(s), zm.sum(0)), (pmm.T @ ac["hm"], pmm.sum(0)), (psm.T @ ac["hm"], psm.sum(0))]
    out["grads"]["actor"], out["gabs"]["actor"] = flat(g), flat(ga)
    new["actor"], new["actor_m"], new["actor_v"] = adam(st["actor"], st["actor_m"], st["actor_v"], out["grads"]["actor"], hp["actor_lr"], t)
    out["evals"] += [ac, q[0], q[1]]
    out["q_gap"] = (np.abs(q1 - q2), 1e-30 + q[0]["qabs"] + q[1]["qabs"])
    # alpha (:371-376): alpha_loss = mean((entropy - target_entropy).detach() * exp(log_alpha))
    ent = np.mean(-ac["logp"])
    out["g_alpha"] = (ent - hp["target_entropy"]) * alpha
    out["ascale"] = np.mean(np.abs(ac["logp"])) * alpha
    new["log_alpha"], new["la_m"], new["la_v"] = adam(st["log_alpha"], st["la_m"], st["la_v"], out["g_alpha"], hp["alpha_lr"], t)
    # soft_update (:145-147) with the updated critics
    for k in ("1", "2"):
        new["t" + k] = st["t" + k] * (1.0 - hp["tau"]) + new["c" + k] * hp["tau"]
    out["losses"] = np.array([out["l_actor"], out["l_c1"], out["l_c2"], out["g_alpha"]])
    return new, out


def near_decision(out, rel=5e-5, ties_ok=False):
    """Rows of the batch for which some ReLU pre-activation of a network evaluated in the update, or q1 - q2 in the actor leg,
    lies within rel x (the sum of its terms' magnitudes) of 0: any fp32-grade evaluation may take the other side there.
    Returns (rows near one in the TD target, the critic update or the actor's trunk -- each depends on its row alone --, rows
    near one in the updated critics of the actor leg -- these depend on the whole batch through the critic step)."""
    an, ct1, ct2, c1, c2, ac, q1, q2 = out["evals"]
    kink = lambda z, za: (np.abs(z) <= rel * za).any(1)                                 # noqa: E731
    near = kink(an["z"], an["zabs"]) | kink(ac["z"], ac["zabs"])
    for c in (ct1, ct2, c1, c2):
        near |= kink(c["z1"], c["z1abs"]) | kink(c["z2"], c["z2abs"])
    near_actor = np.zeros_like(near)
    for c in (q1, q2):
        near_actor |= kink(c["z1"], c["z1abs"]) | kink(c["z2"], c["z2abs"])
    if not ties_ok:
        gap, scale = out["q_gap"]
        near_actor |= (gap <= rel * scale).any(1)
    return near, near_actor


def golden_state(g):
    st = dict(actor=g["sac_actor0"], c1=g["sac_critic_10"], c2=g["sac_critic_20"], t1=g["sac_target_critic_10"], t2=g["sac_target_critic_20"])
    st = {k: np.asarray(v, np.float64) for k, v in st.items()}
    for k in ("actor", "c1", "c2"):
        st[k + "_m"] = np.zeros_like(st[k]); st[k + "_v"] = np.zeros_like(st[k])
    st.update(log_alpha=float(g["sac_log_alpha0"]), la_m=0.0, la_v=0.0, step=0)
    return st


def init_state(rng, obs, hid):
    """nn.Linear-style uniform initialisation (critic_2 independent of critic_1, targets offset from them), float32 values."""
    def lin(n_out, n_in):
        b = 1.0 / np.sqrt(n_in)
        return [rng.uniform(-b, b, n_out * n_in), rng.uniform(-b, b, n_out)]
    f32 = lambda x: np.concatenate(x).astype(np.float32).astype(np.float64)            # noqa: E731
    st = dict(actor=f32(lin(hid, obs) + lin(A, hid) + lin(A, hid)))
    for k in ("c1", "c2"):
        st[k] = f32(lin(hid, obs + A) + lin(hid, hid) + lin(A, hid))
        st["t" + k[1]] = (st[k] + rng.normal(0, 0.01, st[k].size)).astype(np.float32).astype(np.float64)
    for k in ("actor", "c1", "c2"):
        st[k + "_m"] = np.zeros_like(st[k]); st[k + "_v"] = np.zeros_like(st[k])
    st.update(log_alpha=float(np.float32(np.log(0.01))), la_m=0.0, la_v=0.0, step=0)
    return st


def draw_batch(rng, B, obs, bound):
    s = rng.normal(0, 1, (B, obs)).astype(np.float32); s2 = rng.normal(0, 1, (B, obs)).astype(np.float32)
    a = rng.uniform(-bound, bound, (B, A)).astype(np.float32)
    r = rng.normal(0, 1, B).astype(np.float32); d = (rng.uniform(size=B) < 0.2).astype(np.float32)
    e1 = rng.normal(size=(B, A)).astype(np.float32); e2 = rng.normal(size=(B, A)).astype(np.float32)
    return s, a, r, s2, d, e1, e2


def clean_batch(rng, st, B, obs, hid, bound, ties_ok=False):
    """A batch none of whose rows lies within fp32 noise of a decision point of the float64 update from st.  Rows near one
    that depends on the row alone are drawn again whole; then, with the critic step fixed, rows near one in the actor leg get
    fresh eps_cur only (it enters nothing but the actor leg)."""
    batch = list(draw_batch(rng, B, obs, bound))
    for _ in range(40):
        _, out = sac_update64(st, *batch, obs, hid, bound)
        near, near_actor = near_decision(out, ties_ok=ties_ok)
        if near.any():
            for x, y in zip(batch, draw_batch(rng, int(near.sum()), obs, bound)):
                x[near] = y
        elif near_actor.any():
            batch[6][near_actor] = rng.normal(size=(int(near_actor.sum()), A))
        else:
            return batch
    raise AssertionError("could not draw a batch clear of the decision points (%d + %d rows left)" % (near.sum(), near_actor.sum()))


def read_state(S):
    st = {k: S.get_params(role).astype(np.float64)
          for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v"))}
    sc = S.scalars()
    st.update(log_alpha=float(sc["log_alpha"]), la_m=float(sc["la_m"]), la_v=float(sc["la_v"]), step=int(sc["adam_step"]))
    return st


def check_step(S, prev, new, out, losses, what):
    """One update of the learner S (state prev before it) against the float64 step (new, out) computed from prev.

    Bounds (tol_g is a gradient entry's bound: 1e-4 x its magnitude bound from sac_update64 + 1e-4 |g64|; fp32 sums over at
    most 128 terms per dot product and a fixed-order reduction over the batch stay well inside it):
      - losses: actor 1e-5 x mean(|alpha logp| + |min q|) + 1e-4 relative; critics 1e-5 x mean(|Q - y| (|Q| + |y| + 1)) +
        1e-4 relative; d alpha_loss / d log_alpha 1e-5 x alpha mean|logp| + 1e-4 relative;
      - every reduced gradient entry within tol_g;
      - Adam moments: m within 0.1 tol_g, v within 0.001 (2 |g| tol_g + tol_g^2), both + 1e-6 relative;
      - parameters within 1e-6 + 1e-6 |p| + 2 lr min(1, tol_g / |g64|): a gradient well above its noise moves the parameter by
        a well-defined Adam step, one inside it may flip the step's sign.  An exactly zero float64 gradient gets no allowance;
      - targets: tau x the critics' allowance + 1e-6 |t|; log_alpha as a parameter with its gradient's bound."""
    loss_tol = [1e-5 * out["lscale_actor"], 1e-5 * out["lscale_c1"], 1e-5 * out["lscale_c2"], 1e-5 * out["ascale"]]
    err = np.abs(losses - out["losses"]) - (np.array(loss_tol) + 1e-4 * np.abs(out["losses"]))
    assert (err <= 0).all(), (what, "losses", losses, out["losses"])
    got = read_state(S)
    allow = {}
    for role, k in enumerate(("actor", "c1", "c2")):
        g, g64 = S.grads(role).astype(np.float64), out["grads"][k]
        tol = 1e-4 * out["gabs"][k] + 1e-4 * np.abs(g64) + 1e-12
        e = np.abs(g - g64) - tol
        assert (e <= 0).all(), (what, k, "grad", float(e.max()), int(e.argmax()), int((e > 0).sum()), g[e.argmax()], g64[e.argmax()])
        lr = HP["critic_lr"] if k != "actor" else HP["actor_lr"]
        ratio = np.where(g64 != 0, np.minimum(1.0, tol / np.where(g64 != 0, np.abs(g64), 1.0)), 0.0)
        allow[k] = 2 * lr * ratio
        for suffix, bound in (("_m", 0.1 * tol * 1.01), ("_v", 0.001 * (2 * np.abs(g64) * tol + tol * tol) * 1.01)):
            e = np.abs(got[k + suffix] - new[k + suffix]) - (bound + 1e-6 * np.abs(new[k + suffix]) + 1e-30)
            assert (e <= 0).all(), (what, k + suffix, float(e.max()), int(e.argmax()))
        e = np.abs(got[k] - new[k]) - (1e-6 + 1e-6 * np.abs(new[k]) + allow[k])
        assert (e <= 0).all(), (what, k, float(e.max()), int(e.argmax()), int((e > 0).sum()))
    for k in ("1", "2"):
        e = np.abs(got["t" + k] - new["t" + k]) - (1e-6 + 1e-6 * np.abs(new["t" + k]) + HP["tau"] * allow["c" + k])
        assert (e <= 0).all(), (what, "t" + k, float(e.max()), int(e.argmax()))
    ga = abs(out["g_alpha"])
    tol_a = 1e-5 * out["ascale"] + 1e-4 * ga
    la_allow = 1e-6 + 2 * HP["alpha_lr"] * min(1.0, tol_a / ga)
    assert abs(got["log_alpha"] - new["log_alpha"]) <= la_allow, (what, got["log_alpha"], new["log_alpha"])
    assert abs(got["la_m"] - new["la_m"]) <= 0.1 * tol_a + 1e-6 * abs(new["la_m"])
    assert abs(got["la_v"] - new["la_v"]) <= 0.001 * (2 * ga * tol_a + tol_a ** 2) * 1.01 + 1e-6 * abs(new["la_v"])
    assert got["step"] == new["step"]
