"""The float64 SAC restatement (sac_restatement.py) pinned before it judges any kernel: against the reference's own run
(tests/golden/sac_golden.npz) and against the CPU oracle.  No GPU."""
import os

import numpy as np

import oracle as O
from conftest import GOLDEN
from sac_restatement import HP, draw_batch, golden_state, init_state, sac_update64


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
