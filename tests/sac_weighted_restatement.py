"""The prioritised-replay form of the float64 SAC update (include/uavrl.h, the SAC prioritised-replay block), built on the one
float64 restatement of SAC_Trainer.update in sac_restatement.py: only the critic step is restated here, with the importance
weights; the TD target's networks, the actor leg, the alpha step and the soft update are sac_restatement.sac_update64's own."""
import numpy as np

from sac_restatement import HP, A, actor_fwd, adam, critic_bwd, critic_fwd, flat, unpack, sac_update64


def sac_update64_weighted(st, s, a, r, s2, d, eps_next, eps_cur, obs, hid, bound, w, hp=HP):
    """sac_update64 with importance weights w [B]: the critic losses are mean(w_b (Q - y)^2), and out["abs_err"] holds each row's
    priority error e_b = mean_j |min(Q1, Q2)_j - y_j| from the critics before the step (out["abs_err_scale"]: the magnitude of
    its terms).  Everything sac_update64 returns for the critic step is replaced by the weighted step's."""
    f = lambda x: np.asarray(x, np.float64)                                            # noqa: E731
    s, a, r, s2, d, eps_next, w = map(f, (s, a, r, s2, d, eps_next, w))
    nel = float(s.shape[0] * A)
    alpha = np.exp(st["log_alpha"])
    t = st["step"] + 1
    # the TD target (calc_target, :122-131), as sac_update64 forms it
    an = actor_fwd(unpack(st["actor"], "actor", obs, hid), s2, eps_next, bound)
    ct = [critic_fwd(unpack(st[k], "critic", obs, hid), s2, an["act"]) for k in ("t1", "t2")]
    td = r[:, None] + hp["gamma"] * (np.minimum(ct[0]["q"], ct[1]["q"]) - alpha * an["logp"]) * (1.0 - d[:, None])
    tdabs = np.abs(r)[:, None] + hp["gamma"] * (np.maximum(ct[0]["qabs"], ct[1]["qabs"]) + alpha * np.abs(an["logp"]))
    # the weighted critic step (:343-360 with is_weights)
    wc = w[:, None]
    crit, stepped = {}, dict(st)
    for k in ("c1", "c2"):
        P = unpack(st[k], "critic", obs, hid)
        c = critic_fwd(P, s, a)
        diff = c["q"] - td
        g, ga, _, _ = critic_bwd(P, c, 2.0 * wc * diff / nel, 2.0 * wc * (np.abs(diff) + 0.01 * (c["qabs"] + tdabs)) / nel)
        crit[k] = dict(c=c, l=np.mean(wc * diff * diff), lscale=np.mean(wc * np.abs(diff) * (np.abs(c["q"]) + np.abs(td) + 1.0)),
                       g=flat(g), ga=flat(ga))
        stepped[k], crit[k]["m"], crit[k]["v"] = adam(st[k], st[k + "_m"], st[k + "_v"], crit[k]["g"], hp["critic_lr"], t)
    # the rest of the update on the stepped critics: sac_update64 with a critic step of zero length keeps them as they are
    new, out = sac_update64(stepped, s, a, r, s2, d, eps_next, eps_cur, obs, hid, bound, dict(hp, critic_lr=0.0))
    for i, k in enumerate(("c1", "c2")):
        new[k + "_m"], new[k + "_v"] = crit[k]["m"], crit[k]["v"]
        out["l_" + k], out["lscale_" + k] = crit[k]["l"], crit[k]["lscale"]
        out["grads"][k], out["gabs"][k] = crit[k]["g"], crit[k]["ga"]
        out["evals"][3 + i] = crit[k]["c"]
    out["losses"] = np.array([out["l_actor"], out["l_c1"], out["l_c2"], out["g_alpha"]])
    q1, q2 = crit["c1"]["c"], crit["c2"]["c"]
    out["abs_err"] = np.mean(np.abs(np.minimum(q1["q"], q2["q"]) - td), 1)
    out["abs_err_scale"] = np.mean(np.maximum(q1["qabs"], q2["qabs"]) + tdabs, 1)
    return new, out
