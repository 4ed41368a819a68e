"""The float64 restatement of the discrete SAC learner (sac_discrete_restatement.py) against the reference itself:
tests/golden/sac_discrete_golden.npz holds three SAC_Trainer.update calls with IS_Continuous = 0 (make_sac_discrete_golden.py),
the parameters and Adam moments after each at a stratified sample of flat indices covering every tensor.  No GPU."""
import os

import numpy as np

from sac_discrete_restatement import (HP, categorical_pick, golden_state, param_count, pick_margin, sacd_update64, softmax,
                                      unpack, mlp_fwd)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sac_discrete_golden.npz")
OBS, HID, A = 100, 64, 27


def test_restatement_matches_reference_updates():
    g = np.load(GOLDEN)
    assert np.allclose(g["sacd_hparams"], [HP[k] for k in ("actor_lr", "critic_lr", "alpha_lr", "target_entropy", "gamma", "tau")])
    assert g["sacd_actor0"].size == param_count(OBS, HID, A) == 12379
    st = golden_state(g)
    idx = g["sacd_idx"]
    assert idx.size >= 1024 and np.all(np.diff(idx) > 0) and idx[-1] == param_count(OBS, HID, A) - 1
    K = g["sacd_s"].shape[0]
    for k in range(K):
        a = g["sacd_a"][k]
        assert set(a.tolist()) == set(range(A)) and g["sacd_d"][k].any()
        # the actor's probabilities before the step
        p = softmax(mlp_fwd(unpack(st["actor"], OBS, HID, A), g["sacd_s"][k].astype(np.float64))["out"])
        np.testing.assert_allclose(p, g["sacd_probs"][k], rtol=1e-4, atol=1e-7)
        new, out = sacd_update64(st, g["sacd_s"][k], a, g["sacd_r"][k], g["sacd_s2"][k], g["sacd_d"][k], OBS, HID, A)
        np.testing.assert_allclose(out["l_actor"], g["sacd_actor_loss"][k], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(out["l_c1"], g["sacd_critic_1_loss"][k], rtol=1e-5)
        np.testing.assert_allclose(out["l_c2"], g["sacd_critic_2_loss"][k], rtol=1e-5)
        for key, nm in zip(("actor", "c1", "c2", "t1", "t2"), ("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")):
            np.testing.assert_allclose(new[key][idx], g["sacd_" + nm][k], rtol=0, atol=2e-6, err_msg="%s step %d" % (nm, k))
        for key, nm in zip(("actor", "c1", "c2"), ("actor", "critic_1", "critic_2")):
            np.testing.assert_allclose(new[key + "_m"][idx], g["sacd_%s_m" % nm][k], rtol=1e-3, atol=1e-9, err_msg="%s m step %d" % (nm, k))
            np.testing.assert_allclose(new[key + "_v"][idx], g["sacd_%s_v" % nm][k], rtol=1e-3, atol=1e-12, err_msg="%s v step %d" % (nm, k))
        assert abs(new["log_alpha"] - g["sacd_log_alpha"][k]) < 1e-6
        np.testing.assert_allclose(new["la_m"], g["sacd_log_alpha_m"][k], rtol=1e-4)
        np.testing.assert_allclose(new["la_v"], g["sacd_log_alpha_v"][k], rtol=1e-4)
        st = new


def test_checkpoint_keys_and_shapes():
    g = np.load(GOLDEN)
    keys = [str(k) for k in g["sacd_keys"]]
    assert keys == ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"] * 2
    shapes = [tuple(int(x) for x in s if x) for s in g["sacd_shapes"]]
    assert shapes == [(HID, OBS), (HID,), (HID, HID), (HID,), (A, HID), (A,)] * 2


def test_categorical_rule_inverts_the_cdf():
    """On the reference's own probabilities: u on a fine grid picks each k with frequency p_k, fp32 and float64 agree away
    from the boundaries, and rounding that leaves no pick falls back to the last k with p_k > 0."""
    g = np.load(GOLDEN)
    p = g["sacd_probs"][0][:4].astype(np.float64)
    n = 20000
    u = (np.arange(n) + 0.5) / n
    for row in p:
        picks = np.array([categorical_pick(row, x) for x in u])
        freq = np.bincount(picks, minlength=A) / n
        np.testing.assert_allclose(freq, row / row.sum(), atol=2.0 / n)
        for x in u[::97]:
            if pick_margin(row, x) > 1e-5:
                assert categorical_pick(row.astype(np.float32), x, np.float32) == categorical_pick(row, x)
    # u sum(p) never below the total: the last positive entry
    assert categorical_pick(np.array([0.25, 0.75, 0.0, 0.0]), np.nextafter(1.0, 0.0) * 1.0000001) == 1
    assert categorical_pick(np.array([0.5, 0.5, 0.0]), 0.0) == 0
    assert categorical_pick(np.array([0.0, 0.5, 0.5]), 0.0) == 1
