"""SAC (continuous) learner beyond the shipped network (obs 100, hidden 64, action_bound 1) against a float64 restatement of
one SAC_Trainer.update (Trainer/SAC_Trainer.py:122-147, 325-379; BaseClass/BaseCNN.py:459-500): losses, the reduced gradients
of all three networks and every piece of state after each step, at batches of one tile, of ragged tiles, of several tiles
per CTA and of the benchmark's size.  Also: get_action against float64 and the Philox noise it draws, the lockstep replay ring
read back and replayed through the CPU oracle, a ring-sampled update against the same rows given explicitly, two live
learners of different shapes, and the shapes the learner refuses.

The float64 reference is pinned to the reference's own run (tests/golden/sac_golden.npz) and to the CPU oracle before it
judges anything; those two tests need no GPU."""
import os

import numpy as np
import pytest
import torch

import oracle as O
from conftest import GOLDEN

gpu = pytest.mark.gpu
A = 2                                       # action_dim of the UAV task
SMEM_LIMIT = 227 * 1024                     # shared memory one block may use
HP = dict(actor_lr=1e-4, critic_lr=1e-3, alpha_lr=1e-4, target_entropy=1.0, gamma=0.99, tau=0.05)


# ------------------------------------------------------------------ float64 restatement
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


# ------------------------------------------------------------------ the reference pinned before it judges
def golden_state(g):
    st = dict(actor=g["sac_actor0"], c1=g["sac_critic_10"], c2=g["sac_critic_20"], t1=g["sac_target_critic_10"], t2=g["sac_target_critic_20"])
    st = {k: np.asarray(v, np.float64) for k, v in st.items()}
    for k in ("actor", "c1", "c2"):
        st[k + "_m"] = np.zeros_like(st[k]); st[k + "_v"] = np.zeros_like(st[k])
    st.update(log_alpha=float(g["sac_log_alpha0"]), la_m=0.0, la_v=0.0, step=0)
    return st


def test_float64_reference_matches_reference_trainer():
    """The float64 restatement reproduces the reference's own 6 updates (torch fp32, injected noise): actor loss 2e-4
    relative, log_alpha 1e-6, all five networks within 2e-5 at the recorded steps."""
    g = np.load(os.path.join(GOLDEN, "sac_golden.npz"))
    hp = dict(zip(("actor_lr", "critic_lr", "alpha_lr", "target_entropy", "gamma", "tau"), map(float, g["sac_hparams"])))
    st = golden_state(g)
    snap = list(g["sac_snap"])
    names = dict(actor="actor", c1="critic_1", c2="critic_2", t1="target_critic_1", t2="target_critic_2")
    for step in range(g["sac_s"].shape[0]):
        st, out = sac_update64(st, g["sac_s"][step], g["sac_a"][step], g["sac_r"][step], g["sac_s2"][step], g["sac_d"][step],
                               g["sac_eps_next"][step], g["sac_eps_cur"][step], 100, 64, 1.0, hp)
        assert np.isclose(out["l_actor"], g["sac_actor_loss"][step], rtol=2e-4, atol=2e-5), step
        assert abs(st["log_alpha"] - g["sac_log_alpha"][step]) < 1e-6, step
        if step in snap:
            for k, nm in names.items():
                np.testing.assert_allclose(st[k], g["sac_" + nm][snap.index(step)], rtol=0, atol=2e-5, err_msg="%s %d" % (k, step))


def test_float64_reference_matches_oracle():
    """At the shipped shape and at (12, 17, 0.5) the float64 restatement and the CPU oracle (fp32 with float64 dot products)
    agree on 3 updates of a ragged batch: losses 1e-4 relative, parameters 2e-5, log_alpha 1e-6."""
    rng = np.random.default_rng(11)
    for obs, hid, bound in ((100, 64, 1.0), (12, 17, 0.5)):
        B = 200
        st = init_state(rng, obs, hid)
        ora = O.OracleSac(st["actor"], st["c1"], st["c2"], st["t1"], st["t2"], st["log_alpha"], obs_dim=obs, hidden=hid,
                          action_bound=bound, **HP)
        for _ in range(3):
            s, a, r, s2, d, e1, e2 = draw_batch(rng, B, obs, bound)
            st, out = sac_update64(st, s, a, r, s2, d, e1, e2, obs, hid, bound)
            lo, l1, l2 = ora.update(s, a, r, s2, d, e1, e2)
            np.testing.assert_allclose([lo, l1, l2], out["losses"][:3], rtol=1e-4)
            for k in ("actor", "c1", "c2", "t1", "t2"):
                np.testing.assert_allclose(ora.arr[k], st[k], rtol=0, atol=2e-5, err_msg=k)
            assert abs(ora.log_alpha - st["log_alpha"]) < 1e-6


# ------------------------------------------------------------------ data
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


# ------------------------------------------------------------------ shapes
# (obs_dim, hidden, action_bound, accepted): hidden > 64 runs with the gradient-plane stride widened to round_up(hidden, 32)
SHAPES = [
    (100, 64, 1.0, True),       # shipped (config/Trainer.xml)
    (100, 64, 2.5, True),       # action_bound scales the action and the critics' action gradient
    (100, 32, 1.0, True),
    (100, 16, 1.0, True),
    (100, 50, 1.0, True),       # hidden % 4 != 0: zero pad columns in the backward planes
    (12, 17, 0.5, True),        # odd width: the transposed weights keep ld = out (ldw_of's odd branch)
    (124, 64, 1.0, True),       # largest obs_dim: critic input 126, padded by 2
    (60, 72, 1.0, True),        # hidden > 64: gradient planes of stride 96
    (8, 100, 1.0, True),        # hidden > 64: stride 128
    (4, 1, 1.0, True),          # width-1 edge
]
REFUSED = [                     # (obs_dim, hidden, message)
    (98, 64, "obs_dim must be a multiple of 4"),
    (128, 64, "obs_dim must be at most 124"),
    (100, 72, "networks too large for the SMEM-resident SAC kernels"),
    (8, 128, "networks too large for the SMEM-resident SAC kernels"),
]


def shape_id(sh):
    return "obs%d-h%d-bound%g" % sh[:3]


def make_learner(engine, obs, hid, bound, B, st, **kw):
    S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, **HP, **kw)
    load_state(S, st)
    return S


def load_state(S, st):
    for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v")):
        S.set_params(role, st[k])
    S.set_scalars(st["log_alpha"], st["la_m"], st["la_v"], epoch=st["step"], adam_step=st["step"])


def read_state(S):
    st = {k: S.get_params(role).astype(np.float64)
          for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v"))}
    sc = S.scalars()
    st.update(log_alpha=float(sc["log_alpha"]), la_m=float(sc["la_m"]), la_v=float(sc["la_v"]), step=int(sc["adam_step"]))
    return st


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


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


@pytest.fixture(scope="module")
def engine():
    from uavrl_b200 import engine as e
    return e


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@gpu
def test_shape_table(engine):
    """Every row of SHAPES is accepted and fits the 227 KB a block may use; every row of REFUSED is refused with its message,
    before anything is allocated on the device."""
    for obs, hid, bound, ok in SHAPES:
        smem = engine.sac_smem_bytes(obs, hid)
        assert ok and max(smem) <= SMEM_LIMIT, (obs, hid, smem)
        S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound)
        assert S.smem_bytes() == smem
        assert S.P[0] == hid * obs + hid + 2 * (A * hid + A) and S.P[1] == hid * (obs + A) + hid + hid * hid + hid + A * hid + A
        S.close()
    assert any(h > 64 for _, h, _, _ in SHAPES) and any(h % 4 for _, h, _, _ in SHAPES) and any(h % 2 for _, h, _, _ in SHAPES)
    for obs, widest in ((100, 65), (8, 112)):                                          # the limits README states
        assert max(engine.sac_smem_bytes(obs, widest)) <= SMEM_LIMIT < max(engine.sac_smem_bytes(obs, widest + 1))
    for obs, hid, msg in REFUSED:
        if "too large" in msg:
            assert max(engine.sac_smem_bytes(obs, hid)) > SMEM_LIMIT
        else:
            with pytest.raises(engine.UavrlError, match=msg):
                engine.sac_smem_bytes(obs, hid)


@gpu
@pytest.mark.parametrize("obs,hid,msg", REFUSED)
def test_refusal_allocates_nothing(engine, obs, hid, msg):
    """A refused shape raises its message, and the device's free memory is what it was, within 8 MB (a 0.8 GB replay ring is
    requested, so an allocation before the refusal would show)."""
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(engine.UavrlError, match=msg):
        engine.SacLearner(obs_dim=obs, hidden=hid, batch_size=64, replay_capacity=2_000_000, lockstep_envs=1024)
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 8 << 20


@gpu
def test_failed_allocation_frees_everything(engine):
    """A learner whose replay ring cannot be allocated (4.4e14 bytes) fails with the CUDA error, frees what it had already
    allocated (parameters, partials and a 128 MB TD buffer: the free memory is back within 8 MB), and leaves no error behind
    for the next launch."""
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(engine.UavrlError, match="out of memory"):
        engine.SacLearner(batch_size=1 << 24, replay_capacity=1 << 40, lockstep_envs=1024)
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 8 << 20
    S = engine.SacLearner()
    S.init_params(0)
    S.act(torch.zeros((64, 100), device="cuda"))
    torch.cuda.synchronize()
    S.close()


UPDATE_LEGS = {                 # name -> (B, UAVRL_SAC_MAX_CTAS or 0, shapes it runs on: None = all)
    "B64": (64, 0, None),
    "B200": (200, 0, None),                                           # 7 tiles, the last ragged
    "B200-3ctas": (200, 3, None),                                     # 3 + 2 + 2 tiles per CTA: accumulating partials
    "B16384": (16384, 0, [(100, 64, 1.0), (60, 72, 1.0)]),            # the benchmark's batch: 512 tiles, one per CTA
    "B20011": (20011, 0, [(100, 64, 1.0), (60, 72, 1.0)]),            # 626 tiles over the 4 x n_SM CTA cap
}


def update_cases():
    for leg, (_, _, only) in UPDATE_LEGS.items():
        for sh in SHAPES:
            if only is None or sh[:3] in only:
                yield pytest.param(sh, leg, id="%s-%s" % (shape_id(sh), leg))


@gpu
@pytest.mark.parametrize("shape,leg", list(update_cases()))
def test_update_vs_float64(engine, shape, leg, n_sm, monkeypatch):
    """3 consecutive updates (4 at B <= 200) on explicit batches with injected noise; each is checked against the float64
    update from the learner's state before it (check_step states the bounds).  Rows near a ReLU kink or a q1 / q2 decision of
    the float64 update are drawn again."""
    obs, hid, bound, _ = shape
    B, ctas, _ = UPDATE_LEGS[leg]
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))
    if B > 4 * n_sm * 32:
        assert -(-B // 32) > 4 * n_sm                                 # several tiles per CTA on the default grid
    rng = np.random.default_rng(obs * 1000 + hid + B)
    st = init_state(rng, obs, hid)
    S = make_learner(engine, obs, hid, bound, B, st)
    losses = torch.zeros(4, device="cuda")
    for step in range(4 if B <= 200 else 3):
        prev = read_state(S)
        batch = clean_batch(rng, prev, B, obs, hid, bound)
        new, out = sac_update64(prev, *batch, obs, hid, bound)
        s, a, r, s2, d, e1, e2 = batch
        S.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), dev(e1), dev(e2), losses)
        torch.cuda.synchronize()
        check_step(S, prev, new, out, losses.cpu().numpy().astype(np.float64), (leg, step))
    S.close()


@gpu
@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[4], SHAPES[7]], ids=shape_id)
@pytest.mark.parametrize("ctas", [0, 3])
def test_identical_critics_split_ties(engine, shape, ctas, monkeypatch):
    """critic_2 = critic_1 (and their targets and moments): every min(q1, q2) of the actor leg is an exact tie, and the
    gradient goes half to each critic's path (torch's min backward).  Compared with float64 as in test_update_vs_float64."""
    obs, hid, bound, _ = shape
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))
    B = 200
    rng = np.random.default_rng(7 + hid)
    st = init_state(rng, obs, hid)
    for k in ("c2", "t2", "c2_m", "c2_v"):
        st[k] = st[k.replace("2", "1")].copy()
    S = make_learner(engine, obs, hid, bound, B, st)
    losses = torch.zeros(4, device="cuda")
    for step in range(3):
        prev = read_state(S)
        assert np.array_equal(prev["c1"], prev["c2"])
        batch = clean_batch(rng, prev, B, obs, hid, bound, ties_ok=True)
        new, out = sac_update64(prev, *batch, obs, hid, bound)
        assert (out["q_gap"][0] == 0).all()
        S.update_batch(*map(dev, batch), losses=losses)
        torch.cuda.synchronize()
        check_step(S, prev, new, out, losses.cpu().numpy().astype(np.float64), ("ties", step))
    S.close()


# ------------------------------------------------------------------ get_action
@gpu
@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
def test_act_vs_float64(engine, shape, n_sm):
    """get_action with injected noise at n = 1000 and n = 4 x 32 x n_SM + 37 (past the CTA cap): every action within
    bound x (1e-6 + 2e-5 x the sum of |terms| of its head pre-activations) of float64, after rows near a ReLU kink of the
    actor are drawn again."""
    obs, hid, bound, _ = shape
    rng = np.random.default_rng(obs + hid)
    st = init_state(rng, obs, hid)
    S = make_learner(engine, obs, hid, bound, 64, st)
    P = unpack(st["actor"], "actor", obs, hid)
    for n in (1000, 4 * 32 * n_sm + 37):
        s = rng.normal(0, 1, (n, obs)).astype(np.float32)
        eps = rng.normal(size=(n, A)).astype(np.float32)
        for _ in range(30):
            f = actor_fwd(P, s.astype(np.float64), eps.astype(np.float64), bound)
            near = (np.abs(f["z"]) <= 5e-5 * f["zabs"]).any(1)
            if not near.any():
                break
            s[near] = rng.normal(0, 1, (int(near.sum()), obs))
        assert not near.any()
        got = S.act(dev(s), dev(eps)).cpu().numpy().astype(np.float64)
        (_, _), (Wm, bm), (Ws, bs) = P
        scale = f["h"] @ np.abs(Wm).T + np.abs(bm) + (f["h"] @ np.abs(Ws).T + np.abs(bs)) * np.abs(eps)
        err = np.abs(got - f["act"]) - bound * (1e-6 + 2e-5 * scale)
        assert (err <= 0).all(), (n, float(err.max()), np.unravel_index(err.argmax(), err.shape))
    S.close()


@gpu
def test_act_philox_noise_is_standard_normal(engine):
    """Actor weights zero and head biases set so that mu = 0 and sigma = 0.5: atanh(a / bound) / sigma is the noise get_action
    drew.  Over 2 calls x 2^19 rows x 2 components (about 2 x 10^6 draws, fixed seed): each component passes a KS test
    against N(0, 1) at p > 1e-3, mean within 0.005 and std within 0.005 of 0 and 1, |corr| < 0.01 between the two
    components and between consecutive calls."""
    from scipy import stats
    bound, sigma = 2.0, 0.5
    S = engine.SacLearner(action_bound=bound, seed=123)
    p = np.zeros(S.P[0], np.float32)
    bs_off = S.P[0] - A
    p[bs_off:] = np.log(np.expm1(np.arctanh(sigma)))                    # softplus^-1(atanh(sigma)): tanh(softplus(bs)) = sigma
    S.set_params(0, p)
    n = 1 << 19
    obs = torch.zeros((n, 100), device="cuda")
    draws = []
    for _ in range(2):
        a = S.act(obs).cpu().numpy().astype(np.float64)
        assert np.all(np.abs(a) < bound)
        draws.append(np.arctanh(a / bound) / sigma)
    for e in draws:
        for j in range(A):
            x = e[:, j]
            assert stats.kstest(x, "norm").pvalue > 1e-3
            assert abs(x.mean()) < 0.005 and abs(x.std() - 1.0) < 0.005
        assert abs(np.corrcoef(e[:, 0], e[:, 1])[0, 1]) < 0.01
    for j in range(A):
        assert abs(np.corrcoef(draws[0][:, j], draws[1][:, j])[0, 1]) < 0.01
    S.close()


# ------------------------------------------------------------------ the lockstep ring
@gpu
def test_ring_matches_oracle_rollout_and_ring_update(engine, env_golden, env27_golden):
    """sac_train_run without updates until the ring (8 frames of 96 envs) has wrapped twice, reading back every stored
    transition after each 5 iterations: replaying the stored action[:, 0] through the CPU oracle's continuous step gives the
    same states, rewards, dones and next states (as test_lockstep_ring_matches_oracle_rollout).  Then one update sampled
    from the ring through a logical index tape equals, bit for bit, update_batch on the gathered rows in the same order."""
    from gpu_util import assert_obs, city_and_params
    city, params, ocity, oparams = city_and_params(env_golden, env27_golden)
    N, K, cap_frames, B = 96, 64, 8, 256
    env = engine.EnvBatch(city, params, N, max_subgoals=K, auto_reset=False)
    sc = env.make_scenarios(N, seed=6)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    S = engine.SacLearner(batch_size=B, replay_capacity=N * cap_frames, lockstep_envs=N, seed=9, **HP)
    S.init_params(4)
    ob = O.OracleBatch(ocity, oparams, N, K)
    ob.reset(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    rec = {}                                       # iteration -> (s, r, d, s2) of the oracle
    obs = ob.state(want64=True)[1]
    done_its = 0
    for phase in range(4):
        st = engine.sac_train_run(env, S, 5, do_update=False)
        assert st.env_steps == 5 * N and st.updates == 0
        done_its += 5
        count = S.replay_size()
        assert count == min(done_its, cap_frames) * N
        s, a, r, s2, d = S.gather(np.arange(count))
        first = done_its - count // N
        for f in range(count // N):
            it, rows = first + f, slice(f * N, (f + 1) * N)
            if it not in rec:
                assert it == len(rec)
                s0 = obs
                rew, done, _, _, _ = ob.step_(a[rows, 0].astype(np.float64), O.ACT_CONTINUOUS, want_obs=False)
                obs = ob.state(want64=True)[1]
                rec[it] = (s0, rew, done, obs)
            s0, rew, done, s1 = rec[it]
            assert_obs(s[rows], s0, "s it%d" % it)
            np.testing.assert_allclose(r[rows], rew, rtol=1e-5, atol=1e-5)
            assert np.array_equal(d[rows], done), it
            assert_obs(s2[rows], s1, "s2 it%d" % it)
            assert np.all(np.abs(a[rows]) < 1.0)
    assert len(rec) == done_its == 20 and done_its > 2 * cap_frames
    # a ring-sampled update from a logical index tape vs the explicit batch of the same rows
    rng = np.random.default_rng(3)
    count = S.replay_size()
    tape = rng.choice(count, B, replace=False).astype(np.int32)
    s, a, r, s2, d = S.gather(tape.astype(np.int64))
    e1 = rng.normal(size=(B, A)).astype(np.float32); e2 = rng.normal(size=(B, A)).astype(np.float32)
    X = engine.SacLearner(batch_size=B, seed=9, **HP)
    for role in range(11):
        X.set_params(role, S.get_params(role))
    sc0 = S.scalars()
    X.set_scalars(sc0["log_alpha"], sc0["la_m"], sc0["la_v"], sc0["epoch"], sc0["adam_step"])
    l_ring, l_batch = torch.zeros(4, device="cuda"), torch.zeros(4, device="cuda")
    S.update_replay(dev(tape), dev(e1), dev(e2), l_ring)
    X.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), dev(e1), dev(e2), l_batch)
    torch.cuda.synchronize()
    assert np.array_equal(l_ring.cpu().numpy(), l_batch.cpu().numpy())
    for role in range(14):
        assert np.array_equal(S.get_params(role), X.get_params(role)), role
    assert S.scalars() == X.scalars()
    env.close(); S.close(); X.close()


# ------------------------------------------------------------------ two live learners of different shapes
@gpu
def test_two_live_sac_learners(engine):
    """A hidden-64 learner keeps working after a hidden-16 learner is created: its update and get_action equal those of a
    fresh hidden-64 learner bit for bit."""
    batch = [dev(x) for x in draw_batch(np.random.default_rng(0), 200, 100, 1.0)]

    def run(S):
        S.update_batch(*batch)
        act = S.act(batch[0], batch[5]).cpu().numpy()
        return act, [S.get_params(role) for role in range(14)]

    big = engine.SacLearner(batch_size=200); big.init_params(1)
    small = engine.SacLearner(hidden=16, batch_size=200); small.init_params(1)
    got_a, got_p = run(big)
    fresh = engine.SacLearner(batch_size=200); fresh.init_params(1)
    want_a, want_p = run(fresh)
    assert np.array_equal(got_a, want_a)
    for role in range(14):
        assert np.array_equal(got_p[role], want_p[role]), role
    small.close(); big.close(); fresh.close()


@gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tensor-cores", "fp32"])
def test_two_live_dqn_learners(engine, tc):
    """A [64, 64] Q-network learner keeps working after a [64] learner is created: act (Q values and actions) and an update
    equal those of a fresh [64, 64] learner bit for bit, on the tensor-core path and on the fp32 path."""
    rng = np.random.default_rng(5)
    n, B = 5000, 6000
    x = rng.normal(0, 1, (n, 100)).astype(np.float32)
    s, s2 = rng.normal(0, 1, (B, 100)).astype(np.float32), rng.normal(0, 1, (B, 100)).astype(np.float32)
    a = rng.integers(0, 27, B).astype(np.int32); r = rng.normal(size=B).astype(np.float32); d = np.zeros(B, np.float32)

    def make(hidden):
        L = engine.Learner(100, hidden, 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=1000)
        L.init_params(2)
        assert L.set_tensor_cores(tc) == tc
        return L

    def run(L):
        act, q = L.act(dev(x), 0.0, want_q=True)
        loss = torch.zeros(1, device="cuda")
        L.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), loss)
        return act.cpu().numpy(), q.cpu().numpy(), float(loss), L.get_params(0)

    big = make([64, 64])
    small = make([64])
    got = run(big)
    fresh = make([64, 64])
    want = run(fresh)
    for g_, w_ in zip(got, want):
        assert np.array_equal(g_, w_)
    big.close(); small.close(); fresh.close()
