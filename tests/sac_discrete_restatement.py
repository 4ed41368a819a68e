"""Float64 restatement of the discrete SAC learner (include/uavrl.h, "SAC, discrete actions"; SAC_Trainer.update :380-430
with PolicyNet_SAC / QValueNet_SAC), of its categorical draw, and the helpers its tests share."""
import numpy as np

HP = dict(actor_lr=1e-4, critic_lr=1e-3, alpha_lr=1e-4, target_entropy=1.0, gamma=0.99, tau=0.05)
NETS = ("actor", "c1", "c2", "t1", "t2")


def unpack(p, obs, hid, A):
    """flat state_dict-ordered parameters -> [(W, b)] of fc1, fc2, fc3"""
    out, o = [], 0
    for n_out, n_in in ((hid, obs), (hid, hid), (A, hid)):
        W = p[o:o + n_out * n_in].reshape(n_out, n_in); o += n_out * n_in
        out.append((W, p[o:o + n_out])); o += n_out
    assert o == p.size
    return out


def param_count(obs, hid, A):
    return hid * obs + hid + hid * hid + hid + A * hid + A


def mlp_fwd(P, x):
    """fc1 -> ReLU -> fc2 -> ReLU -> fc3, with each pre-activation's magnitude bound (the sum of its terms' |.|)"""
    (W1, b1), (W2, b2), (W3, b3) = P
    z1 = x @ W1.T + b1; z1abs = np.abs(x) @ np.abs(W1).T + np.abs(b1)
    h1 = np.maximum(z1, 0.0); h1m = np.where(z1 > 0, z1abs, 0.0)
    z2 = h1 @ W2.T + b2; z2abs = h1m @ np.abs(W2).T + np.abs(b2)
    h2 = np.maximum(z2, 0.0); h2m = np.where(z2 > 0, z2abs, 0.0)
    out = h2 @ W3.T + b3; outabs = h2m @ np.abs(W3).T + np.abs(b3)
    return dict(x=x, z1=z1, z1abs=z1abs, h1=h1, h1m=h1m, z2=z2, z2abs=z2abs, h2=h2, h2m=h2m, out=out, outabs=outabs)


def mlp_bwd(P, f, dout, dabs):
    """flat parameter gradient of sum(dout * out) and its magnitude bound (the same chain on |.|)"""
    (W1, _), (W2, _), (W3, _) = P
    d2 = (dout @ W3) * (f["z2"] > 0); a2 = (dabs @ np.abs(W3)) * (f["z2"] > 0)
    d1 = (d2 @ W2) * (f["z1"] > 0); a1 = (a2 @ np.abs(W2)) * (f["z1"] > 0)
    g = [d1.T @ f["x"], d1.sum(0), d2.T @ f["h1"], d2.sum(0), dout.T @ f["h2"], dout.sum(0)]
    ga = [a1.T @ np.abs(f["x"]), a1.sum(0), a2.T @ f["h1m"], a2.sum(0), dabs.T @ f["h2m"], dabs.sum(0)]
    return np.concatenate([x.ravel() for x in g]), np.concatenate([x.ravel() for x in ga])


def softmax(z):
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def adam(p, m, v, g, lr, t):
    """torch.optim.Adam's single-tensor step in the form reduce_adam_kernel computes it"""
    bc1, bc2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
    m = m + (g - m) * 0.1
    v = v * 0.999 + 0.001 * g * g
    return p - (lr / bc1) * (m / (np.sqrt(v) / np.sqrt(bc2) + 1e-8)), m, v


def policy_terms(p, q1, q2, alpha):
    """per row: H = -sum p log(p + 1e-8), m = sum p min(Q1, Q2)"""
    lp = np.log(p + 1e-8)
    mn = np.minimum(q1, q2)
    return -(p * lp).sum(1), (p * mn).sum(1), lp, mn


def sacd_update64(st, s, a, r, s2, d, obs, hid, A, hp=HP):
    """One discrete SAC_Trainer.update in float64 from state st (actor, c1, c2, t1, t2, their Adam moments, log_alpha, la_m,
    la_v, step).  Returns (new state, out): out holds the four loss outputs, the three reduced gradients with their
    magnitude bounds, the actor's probabilities on s and the forward passes (for the decision-point checks)."""
    f = lambda x: np.asarray(x, np.float64)                                            # noqa: E731
    s, r, s2, d = map(f, (s, r, s2, d))
    a = np.asarray(a, np.int64)
    B = s.shape[0]
    t = st["step"] + 1
    new = dict(st, step=t)
    alpha = np.exp(st["log_alpha"])
    Pa = unpack(st["actor"], obs, hid, A)
    Pc = [unpack(st[k], obs, hid, A) for k in ("c1", "c2", "t1", "t2")]
    rr = (r + 10.0) / 10.0                                                             # reward shaping (:390)
    # calc_target (:133-141)
    an = mlp_fwd(Pa, s2)
    pn = softmax(an["out"])
    ct = [mlp_fwd(Pc[2], s2), mlp_fwd(Pc[3], s2)]
    Hn, mn, lpn, _ = policy_terms(pn, ct[0]["out"], ct[1]["out"], alpha)
    y = rr + hp["gamma"] * (mn + alpha * Hn) * (1.0 - d)
    yabs = np.abs(rr) + hp["gamma"] * ((pn * np.maximum(ct[0]["outabs"], ct[1]["outabs"])).sum(1) + alpha * np.abs(Hn) + 1e-7)
    out = dict(evals=[an, ct[0], ct[1]], grads={}, gabs={})
    rows = np.arange(B)
    # critics (:397-406)
    for i, k in enumerate(("c1", "c2")):
        c = mlp_fwd(Pc[i], s)
        q = c["out"][rows, a]
        diff = q - y
        out["l_" + k] = np.mean(diff * diff)
        out["lscale_" + k] = np.mean(np.abs(diff) * (c["outabs"][rows, a] + yabs + 1.0))
        dq = np.zeros((B, A)); dqa = np.zeros((B, A))
        dq[rows, a] = 2.0 * diff / B
        dqa[rows, a] = 2.0 * (np.abs(diff) + 0.01 * (c["outabs"][rows, a] + yabs)) / B
        out["grads"][k], out["gabs"][k] = mlp_bwd(Pc[i], c, dq, dqa)
        new[k], new[k + "_m"], new[k + "_v"] = adam(st[k], st[k + "_m"], st[k + "_v"], out["grads"][k], hp["critic_lr"], t)
        out["evals"].append(c)
    # actor (:408-419) on the updated critics
    Pn = [unpack(new[k], obs, hid, A) for k in ("c1", "c2")]
    q = [mlp_fwd(Pn[0], s), mlp_fwd(Pn[1], s)]
    ac = mlp_fwd(Pa, s)
    p = softmax(ac["out"])
    H, m, lp, mnq = policy_terms(p, q[0]["out"], q[1]["out"], alpha)
    out["probs"] = p
    out["l_actor"] = np.mean(-alpha * H - m)
    mabs = np.maximum(q[0]["outabs"], q[1]["outabs"])
    out["lscale_actor"] = np.mean(alpha * np.abs(H) + (p * mabs).sum(1))
    g = (alpha * (lp + p / (p + 1e-8)) - mnq) / B
    gab = (alpha * (np.abs(lp) + 1.0) + mabs) / B
    dz = p * (g - (p * g).sum(1, keepdims=True))
    dza = p * (gab + (p * gab).sum(1, keepdims=True))
    out["grads"]["actor"], out["gabs"]["actor"] = mlp_bwd(Pa, ac, dz, dza)
    new["actor"], new["actor_m"], new["actor_v"] = adam(st["actor"], st["actor_m"], st["actor_v"], out["grads"]["actor"], hp["actor_lr"], t)
    out["evals"] += [ac, q[0], q[1]]
    # alpha: mean((H - target_entropy) alpha), the gradient with respect to log_alpha
    out["g_alpha"] = (np.mean(H) - hp["target_entropy"]) * alpha
    out["ascale"] = (np.mean(np.abs(H)) + 1.0) * alpha
    new["log_alpha"], new["la_m"], new["la_v"] = adam(st["log_alpha"], st["la_m"], st["la_v"], out["g_alpha"], hp["alpha_lr"], t)
    for k in ("1", "2"):
        new["t" + k] = st["t" + k] * (1.0 - hp["tau"]) + new["c" + k] * hp["tau"]
    out["losses"] = np.array([out["l_actor"], out["l_c1"], out["l_c2"], out["g_alpha"]])
    return new, out


def categorical_pick(p, u, dtype=np.float64):
    """The device draw on one row: the smallest k with u sum(p) < p_0 + ... + p_k (summed left to right in `dtype`), else the
    last k with p_k > 0."""
    p = np.asarray(p, dtype)
    s = dtype(0)
    for x in p:
        s = dtype(s + x)
    t = dtype(dtype(u) * s)
    c = dtype(0)
    for k, x in enumerate(p):
        c = dtype(c + x)
        if t < c:
            return k
    nz = np.nonzero(p > 0)[0]
    return int(nz[-1]) if nz.size else p.size - 1


def pick_margin(p, u):
    """distance of u sum(p) from the nearest cumulative boundary, relative to sum(p): below ~1e-5 an fp32 draw may differ"""
    c = np.cumsum(np.asarray(p, np.float64))
    return np.min(np.abs(u * c[-1] - c)) / c[-1]


def near_kink(out, rel=5e-5):
    """rows with a ReLU pre-activation within rel x its magnitude of 0 in a forward pass the update back-propagates through
    (both critics and the actor on s, with the parameters before the step): an fp32 evaluation may take the other side there,
    which switches a whole gradient row on or off.  The forward-only passes (the target's three networks, the updated critics
    of the actor leg) only move a value by about the pre-activation itself there, well inside the bounds."""
    kink = lambda f: ((np.abs(f["z1"]) <= rel * f["z1abs"]).any(1) | (np.abs(f["z2"]) <= rel * f["z2abs"]).any(1))  # noqa: E731
    _, _, _, c1, c2, ac, _, _ = out["evals"]
    return kink(c1) | kink(c2) | kink(ac)


def init_state(rng, obs, hid, A):
    """nn.Linear-style uniform initialisation, float32 values; targets offset from the critics"""
    def lin(n_out, n_in):
        b = 1.0 / np.sqrt(n_in)
        return [rng.uniform(-b, b, n_out * n_in), rng.uniform(-b, b, n_out)]
    f32 = lambda x: np.concatenate(x).astype(np.float32).astype(np.float64)            # noqa: E731
    st = {}
    for k in ("actor", "c1", "c2"):
        st[k] = f32(lin(hid, obs) + lin(hid, hid) + lin(A, hid))
    for k in ("1", "2"):
        st["t" + k] = (st["c" + k] + rng.normal(0, 0.01, st["c" + k].size)).astype(np.float32).astype(np.float64)
    for k in ("actor", "c1", "c2"):
        st[k + "_m"] = np.zeros_like(st[k]); st[k + "_v"] = np.zeros_like(st[k])
    st.update(log_alpha=float(np.float32(np.log(0.01))), la_m=0.0, la_v=0.0, step=0)
    return st


def golden_state(g):
    """the recorded initial state; the targets start as copies of the critics (SAC_Trainer.py:33-34)"""
    st = {k: np.asarray(g["sacd_%s0" % nm], np.float64) for k, nm in (("actor", "actor"), ("c1", "critic_1"), ("c2", "critic_2"))}
    st["t1"], st["t2"] = st["c1"].copy(), st["c2"].copy()
    for k in ("actor", "c1", "c2"):
        st[k + "_m"] = np.zeros_like(st[k]); st[k + "_v"] = np.zeros_like(st[k])
    st.update(log_alpha=float(g["sacd_log_alpha0"]), la_m=0.0, la_v=0.0, step=0)
    return st


def draw_batch(rng, B, obs, A):
    s = rng.normal(0, 1, (B, obs)).astype(np.float32); s2 = rng.normal(0, 1, (B, obs)).astype(np.float32)
    a = rng.integers(0, A, B).astype(np.int32)
    if B >= A:
        a[:A] = np.arange(A)
    r = rng.normal(-2, 6, B).astype(np.float32); d = (rng.uniform(size=B) < 0.2).astype(np.float32)
    return [s, a, r, s2, d]


def clean_batch(rng, st, B, obs, hid, A):
    """A batch none of whose rows lies within fp32 noise of a ReLU kink that the float64 update from st back-propagates
    through; such a row depends on itself alone, so it is drawn again whole."""
    batch = draw_batch(rng, B, obs, A)
    for _ in range(60):
        _, out = sacd_update64(st, *batch, obs, hid, A)
        bad = near_kink(out)
        if not bad.any():
            return batch
        for x, y in zip(batch, draw_batch(rng, int(bad.sum()), obs, A)):
            x[bad] = y
    raise AssertionError("could not draw a batch clear of the ReLU kinks (%d rows left)" % bad.sum())


def read_state(S):
    st = {k: S.get_params(role).astype(np.float64)
          for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v"))}
    sc = S.scalars()
    st.update(log_alpha=float(sc["log_alpha"]), la_m=float(sc["la_m"]), la_v=float(sc["la_v"]), step=int(sc["adam_step"]))
    return st


def check_step(S, new, out, losses, what, hp=HP):
    """One update of the learner S against the float64 step (new, out) computed from its state before.  Bounds, with tol_g an
    entry's gradient bound 1e-4 x its magnitude bound + 1e-4 |g64|:
      - losses within 1e-5 x their magnitude scale + 1e-4 relative;
      - every reduced gradient entry within tol_g; Adam m within 0.1 tol_g and v within 0.001 (2 |g| tol_g + tol_g^2);
      - parameters within 1e-6 + 1e-6 |p| + 2 lr min(1, tol_g / |g64|) (a gradient inside its noise may flip the step's
        sign); targets within tau x that; log_alpha likewise with its gradient's bound."""
    loss_tol = np.array([out["lscale_actor"], out["lscale_c1"], out["lscale_c2"], out["ascale"]]) * 1e-5
    err = np.abs(losses - out["losses"]) - (loss_tol + 1e-4 * np.abs(out["losses"]))
    assert (err <= 0).all(), (what, "losses", losses, out["losses"])
    got = read_state(S)
    allow = {}
    for role, k in enumerate(("actor", "c1", "c2")):
        g, g64 = S.grads(role).astype(np.float64), out["grads"][k]
        tol = 1e-4 * out["gabs"][k] + 1e-4 * np.abs(g64) + 1e-12
        e = np.abs(g - g64) - tol
        assert (e <= 0).all(), (what, k, "grad", float(e.max()), int(e.argmax()), int((e > 0).sum()), g[e.argmax()], g64[e.argmax()])
        lr = hp["critic_lr"] if k != "actor" else hp["actor_lr"]
        ratio = np.where(g64 != 0, np.minimum(1.0, tol / np.where(g64 != 0, np.abs(g64), 1.0)), 0.0)
        allow[k] = 2 * lr * ratio
        for suffix, bound in (("_m", 0.1 * tol * 1.01), ("_v", 0.001 * (2 * np.abs(g64) * tol + tol * tol) * 1.01)):
            e = np.abs(got[k + suffix] - new[k + suffix]) - (bound + 1e-6 * np.abs(new[k + suffix]) + 1e-30)
            assert (e <= 0).all(), (what, k + suffix, float(e.max()), int(e.argmax()))
        e = np.abs(got[k] - new[k]) - (1e-6 + 1e-6 * np.abs(new[k]) + allow[k])
        assert (e <= 0).all(), (what, k, float(e.max()), int(e.argmax()), int((e > 0).sum()))
    for k in ("1", "2"):
        e = np.abs(got["t" + k] - new["t" + k]) - (1e-6 + 1e-6 * np.abs(new["t" + k]) + hp["tau"] * allow["c" + k])
        assert (e <= 0).all(), (what, "t" + k, float(e.max()), int(e.argmax()))
    ga = abs(out["g_alpha"])
    tol_a = 1e-5 * out["ascale"] + 1e-4 * ga
    la_allow = 1e-6 + 2 * hp["alpha_lr"] * min(1.0, tol_a / max(ga, 1e-30))
    assert abs(got["log_alpha"] - new["log_alpha"]) <= la_allow, (what, got["log_alpha"], new["log_alpha"])
