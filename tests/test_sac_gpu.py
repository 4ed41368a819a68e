"""SAC continuous on the GPU (through the C ABI) against the reference's SAC_Trainer (golden vectors with injected
reparameterisation noise) and the CPU oracle.  Tolerance: parameters of actor / critics / targets 2e-5 (abs) after
6 updates, log_alpha 1e-6, losses 2e-4 relative; get_action samples 2e-6."""
import os

import numpy as np
import pytest
import torch

import oracle as O
from conftest import GOLDEN
from gpu_util import city_and_params, dev

pytestmark = pytest.mark.gpu


def load(S, g):
    for role, nm in enumerate(("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")):
        S.set_params(role, g["sac_%s0" % nm])
    S.set_scalars(float(g["sac_log_alpha0"]))


def test_sac_update_matches_reference_trainer():
    from uavrl_b200 import engine
    g = np.load(os.path.join(GOLDEN, "sac_golden.npz"))
    hp = g["sac_hparams"]
    S = engine.SacLearner(actor_lr=hp[0], critic_lr=hp[1], alpha_lr=hp[2], target_entropy=hp[3], gamma=hp[4], tau=hp[5], batch_size=64)
    assert S.P == [6724, 10882, 10882, 10882, 10882]
    load(S, g)
    ora = O.OracleSac(g["sac_actor0"], g["sac_critic_10"], g["sac_critic_20"], g["sac_target_critic_10"], g["sac_target_critic_20"],
                      float(g["sac_log_alpha0"]), actor_lr=hp[0], critic_lr=hp[1], alpha_lr=hp[2], target_entropy=hp[3], gamma=hp[4], tau=hp[5])
    snap = list(g["sac_snap"])
    losses = torch.zeros(4, device="cuda")
    for step in range(g["sac_s"].shape[0]):
        S.update_batch(dev(g["sac_s"][step]), dev(g["sac_a"][step]), dev(g["sac_r"][step]), dev(g["sac_s2"][step]), dev(g["sac_d"][step]),
                       dev(g["sac_eps_next"][step]), dev(g["sac_eps_cur"][step]), losses)
        lo, l1, l2 = ora.update(g["sac_s"][step], g["sac_a"][step], g["sac_r"][step], g["sac_s2"][step], g["sac_d"][step],
                                g["sac_eps_next"][step], g["sac_eps_cur"][step])
        torch.cuda.synchronize()
        got = losses.cpu().numpy()
        assert np.isclose(got[0], g["sac_actor_loss"][step], rtol=2e-4, atol=2e-5), (step, got[0])
        assert np.isclose(got[1], l1, rtol=2e-4) and np.isclose(got[2], l2, rtol=2e-4), (step, got, l1, l2)
        sc = S.scalars()
        assert abs(sc["log_alpha"] - g["sac_log_alpha"][step]) < 1e-6 and sc["epoch"] == step + 1 == sc["adam_step"]
        if step in snap:
            k = snap.index(step)
            for role, nm in enumerate(("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")):
                np.testing.assert_allclose(S.get_params(role), g["sac_" + nm][k], rtol=0, atol=2e-5, err_msg="%s step %d" % (nm, step))
    # get_action on the final actor with injected noise (SAC_Trainer.py:444-448)
    a = S.act(dev(g["sac_s"][0][:8]), dev(g["sac_act_eps"])).cpu().numpy()
    np.testing.assert_allclose(a, g["sac_act_out"], rtol=0, atol=2e-6)
    S.close()


@pytest.mark.parametrize("max_ctas", [0, 3])
def test_sac_ragged_batch_vs_oracle_and_philox_noise(max_ctas, monkeypatch):
    """max_ctas = 3: 7 tiles on 3 persistent CTAs (3 + 2 + 2 tiles) -- the accumulating multi-tile path every batch above
    32 x #SMs samples takes (BASELINE configs[4]: 16 384 samples = 512 tiles on 132 CTAs)."""
    from uavrl_b200 import engine
    if max_ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(max_ctas))
    g = np.load(os.path.join(GOLDEN, "sac_golden.npz"))
    rng = np.random.default_rng(2)
    B = 200                                         # not a multiple of the 32-sample tile
    s = np.tile(g["sac_s"].reshape(-1, 100), (2, 1))[:B]; s2 = np.tile(g["sac_s2"].reshape(-1, 100), (2, 1))[:B]
    a = rng.uniform(-1, 1, (B, 2)).astype(np.float32); r = rng.normal(0, 1, B).astype(np.float32)
    d = (rng.uniform(size=B) < 0.2).astype(np.float32)
    e1 = rng.normal(size=(B, 2)).astype(np.float32); e2 = rng.normal(size=(B, 2)).astype(np.float32)
    S = engine.SacLearner(batch_size=B)
    load(S, g)
    ora = O.OracleSac(g["sac_actor0"], g["sac_critic_10"], g["sac_critic_20"], g["sac_target_critic_10"], g["sac_target_critic_20"],
                      float(g["sac_log_alpha0"]))
    for _ in range(3):
        S.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), dev(e1), dev(e2))
        ora.update(s, a, r, s2, d, e1, e2)
    for role, nm in enumerate(("actor", "c1", "c2", "t1", "t2")):
        np.testing.assert_allclose(S.get_params(role), ora.arr[nm], rtol=0, atol=2e-5, err_msg=nm)
    assert abs(S.scalars()["log_alpha"] - ora.log_alpha) < 1e-6
    # Philox noise path: actions in (-1, 1), roughly centred on tanh(mu), different between calls
    obs = dev(s)
    a1 = S.act(obs).cpu().numpy(); a2 = S.act(obs).cpu().numpy()
    assert np.all(np.abs(a1) < 1) and not np.array_equal(a1, a2)
    mean_noise = np.mean([S.act(obs).cpu().numpy() for _ in range(64)], axis=0)
    a0, _ = ora.actor_forward(s, np.zeros((B, 2), np.float32))
    assert np.abs(mean_noise - a0).mean() < 0.1
    S.close()


def test_sac_lockstep_loop_with_reference_continuous_step(env_golden, env27_golden):
    """The reference's own shipped configuration (SAC + continuous update_PathPlan), N envs in lockstep."""
    from uavrl_b200 import engine
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N = 256
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(512, seed=5)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    S = engine.SacLearner(batch_size=N, replay_capacity=N * 32, lockstep_envs=N, seed=3)
    S.init_params(2)
    p0 = S.get_params(0)
    st = engine.sac_train_run(env, S, 120)
    assert st.env_steps == 120 * N and st.updates == 119
    assert np.isfinite(st.last_loss) and np.isfinite(st.sum_reward) and st.n_success >= N      # first step of every episode is a 'success'
    p1 = S.get_params(0)
    assert np.isfinite(p1).all() and np.abs(p1 - p0).max() > 1e-4
    sc2 = S.scalars()
    assert sc2["epoch"] == 120 and sc2["adam_step"] == 119 and np.isfinite(sc2["log_alpha"])
    for r in (3, 4):
        assert np.isfinite(S.get_params(r)).all()
    env.close(); S.close()
