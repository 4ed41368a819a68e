"""Discrete SAC on the GPU (SacLearner(discrete=True), include/uavrl.h "SAC, discrete actions"): the update against the
reference's own SAC_Trainer (golden vectors, the continuous golden test's tolerances) and a shape sweep against the float64
restatement; the categorical draw; the lockstep loop on the 27-action step; grouped trainers; the refusals."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

import replay_restatement as R
from conftest import GOLDEN
from gpu_util import assert_same, city_and_params, dev
from sac_discrete_restatement import (HP, categorical_pick, clean_batch, init_state, pick_margin, read_state, sacd_update64, set_state,
                                      softmax, unpack, mlp_fwd, check_step)

pytestmark = pytest.mark.gpu
SMEM_MAX = 232448
NETS = ("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")


def engine():
    from uavrl_b200 import engine as E
    return E


def sacd(obs=100, hid=64, A=27, **kw):
    kw.setdefault("batch_size", 64)
    return engine().SacLearner(obs_dim=obs, hidden=hid, act_dim=A, discrete=True, **HP, **kw)


def widest_hidden(obs, A):
    """the widest hidden layer whose four kernels fit 227 KB of shared memory"""
    best = 0
    for h in range(1, 129):
        if max(engine().sac_smem_bytes(obs, h, 0, A, True)) <= SMEM_MAX:
            best = h
    return best


# ------------------------------------------------------------------ the update
def test_update_matches_reference_trainer():
    g = np.load(os.path.join(GOLDEN, "sac_discrete_golden.npz"))
    hp = g["sacd_hparams"]
    S = engine().SacLearner(hidden=64, act_dim=27, discrete=True, actor_lr=hp[0], critic_lr=hp[1], alpha_lr=hp[2],
                            target_entropy=hp[3], gamma=hp[4], tau=hp[5], batch_size=64)
    assert S.P == [12379] * 5
    assert [k for k, _ in S.layout(0)] == [str(k) for k in g["sacd_keys"][:6]]
    idx = g["sacd_idx"]                                  # the reference's parameters after each step are kept at these entries
    for role, nm in enumerate(("actor", "critic_1", "critic_2", "critic_1", "critic_2")):   # the targets start as the critics
        S.set_params(role, g["sacd_%s0" % nm])
    S.set_scalars(float(g["sacd_log_alpha0"]))
    losses = torch.zeros(4, device="cuda")
    for k in range(g["sacd_s"].shape[0]):
        S.update_batch(dev(g["sacd_s"][k]), dev(g["sacd_a"][k]), dev(g["sacd_r"][k]), dev(g["sacd_s2"][k]), dev(g["sacd_d"][k]),
                       losses=losses)
        torch.cuda.synchronize()
        got = losses.cpu().numpy()
        assert np.isclose(got[0], g["sacd_actor_loss"][k], rtol=2e-4, atol=2e-5), (k, got[0], g["sacd_actor_loss"][k])
        assert np.isclose(got[1], g["sacd_critic_1_loss"][k], rtol=2e-4) and np.isclose(got[2], g["sacd_critic_2_loss"][k], rtol=2e-4), (k, got)
        sc = S.scalars()
        assert abs(sc["log_alpha"] - g["sacd_log_alpha"][k]) < 1e-6 and sc["epoch"] == k + 1 == sc["adam_step"]
        for role, nm in enumerate(NETS):
            np.testing.assert_allclose(S.get_params(role)[idx], g["sacd_" + nm][k], rtol=0, atol=2e-5, err_msg="%s step %d" % (nm, k))
    S.close()


def sweep_rows():
    rows = [(27, 64, 100, B) for B in (1, 31, 32, 33, 64, 4096)]
    rows += [(2, 1, 4, 33), (31, 32, 128, 64), (2, 64, 100, 31), (31, 1, 100, 32), (27, 32, 4, 1), (2, 32, 128, 4096)]
    rows += [(A, "widest", obs, 64) for A in (2, 27, 31) for obs in (4, 100, 128)]
    return rows


@pytest.mark.parametrize("A,hid,obs,B", sweep_rows())
def test_update_shape_sweep(A, hid, obs, B):
    """Two updates on batches clear of the ReLU kinks of the float64 step, each checked entry by entry against it."""
    if hid == "widest":
        hid = widest_hidden(obs, A)
        assert hid >= 32
    rng = np.random.default_rng(A * 1000 + obs + hid + B)
    S = sacd(obs, hid, A, batch_size=B)
    assert max(S.smem_bytes()) <= SMEM_MAX
    st = init_state(rng, obs, hid, A)
    set_state(S, st)
    losses = torch.zeros(4, device="cuda")
    for step in range(2):
        batch = clean_batch(rng, st, B, obs, hid, A)
        new, out = sacd_update64(st, *batch, obs, hid, A)
        s, a, r, s2, d = batch
        S.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), losses=losses)
        torch.cuda.synchronize()
        check_step(S, new, out, losses.cpu().numpy().astype(np.float64), (A, hid, obs, B, step))
        st = read_state(S)
    S.close()


def test_update_accumulates_tiles_on_few_ctas(monkeypatch):
    """UAVRL_SAC_MAX_CTAS = 3: 7 tiles on 3 CTAs, the accumulating path every batch above 4 x 32 x #SMs takes."""
    monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", "3")
    rng = np.random.default_rng(5)
    S = sacd(batch_size=200)
    st = init_state(rng, 100, 64, 27)
    set_state(S, st)
    batch = clean_batch(rng, st, 200, 100, 64, 27)
    new, out = sacd_update64(st, *batch, 100, 64, 27)
    losses = torch.zeros(4, device="cuda")
    S.update_batch(*(dev(x) for x in batch), losses=losses)
    torch.cuda.synchronize()
    check_step(S, new, out, losses.cpu().numpy().astype(np.float64), "max_ctas 3")
    S.close()


# ------------------------------------------------------------------ get_action
def probs_of(st, obs_rows, obs, hid, A):
    return softmax(mlp_fwd(unpack(st["actor"], obs, hid, A), obs_rows.astype(np.float64))["out"])


@pytest.mark.parametrize("A,obs,hid", [(27, 100, 64), (2, 4, 1), (31, 128, 32)])
def test_act_tape_philox_and_argmax(A, obs, hid):
    rng = np.random.default_rng(A + obs)
    S = sacd(obs, hid, A)
    st = init_state(rng, obs, hid, A)
    st["actor"][-A:] += rng.normal(0, 2, A)            # spread the probabilities
    set_state(S, st)
    n = 1000
    x = rng.normal(0, 1, (n, obs)).astype(np.float32)
    p = probs_of(st, x, obs, hid, A)
    u = rng.uniform(size=n).astype(np.float32)
    a = S.act(dev(x), u=dev(u)).cpu().numpy()
    ok = np.array([pick_margin(p[i], u[i]) > 1e-5 for i in range(n)])
    want = np.array([categorical_pick(p[i], u[i]) for i in range(n)])
    assert ok.mean() > 0.95 and np.array_equal(a[ok], want[ok])
    # the Philox stream: word 0 of Philox(key of seed, 2^63 | act call, row); the tape's call above was call 0
    for call in (1, 2):
        a = S.act(dev(x)).cpu().numpy()
        uu = R.u01(R.philox(R.trainer_key(42 ^ R.K_NOISE_SALT, R.K_NOISE_SALT, 0), R.SAC_ACT_CTR | call, np.arange(n))[:, 0])
        ok = np.array([pick_margin(p[i], uu[i]) > 1e-5 for i in range(n)])
        want = np.array([categorical_pick(p[i], uu[i]) for i in range(n)])
        assert ok.mean() > 0.95 and np.array_equal(a[ok], want[ok]), call
    # argmax p, drawing nothing
    srt = np.sort(p, 1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-5 * srt[:, -1]
    m = S.act(dev(x), mean=True).cpu().numpy()
    assert np.array_equal(m[clear], p.argmax(1)[clear])
    S.close()


def test_act_frequencies_chi_square():
    """One seeded 1 M-row draw at fixed probabilities (fc3 weights zero, its bias the log-probabilities)."""
    rng = np.random.default_rng(77)
    A, n = 27, 1 << 20
    S = sacd(seed=1234)
    st = init_state(rng, 100, 64, A)
    p = rng.dirichlet(np.ones(A) * 0.7)
    p[3] = 0.0                                            # an impossible action is never drawn
    p /= p.sum()
    st["actor"][-A - A * 64:-A] = 0.0
    st["actor"][-A:] = np.log(np.maximum(p, 1e-30))
    set_state(S, st)
    x = torch.zeros((n, 100), device="cuda")
    a = S.act(x).cpu().numpy()
    counts = np.bincount(a, minlength=A)
    assert counts[3] == 0 and a.min() >= 0 and a.max() < A
    keep = p > 0
    chi2 = (((counts - n * p) ** 2)[keep] / (n * p[keep])).sum()
    assert stats.chi2.sf(chi2, keep.sum() - 1) > 1e-4, chi2
    S.close()


# ------------------------------------------------------------------ the lockstep loop
@pytest.fixture(scope="module")
def world(env_golden, env27_golden):
    return city_and_params(env_golden, env27_golden)[:2]


def make_env(world, N, seed=8):
    city, params = world
    env = engine().EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(1024, seed=seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    return env


def twin(S, B, G=1, seed=9):
    X = sacd(batch_size=B, seed=seed, trainers=G)
    for role in range(11):
        X.set_params(role, S.get_params(role))
    sc = S.scalars()
    X.set_scalars(sc["log_alpha"], sc["la_m"], sc["la_v"], sc["epoch"], sc["adam_step"])
    X.set_alpha(S.alpha())
    return X


@pytest.mark.parametrize("G", [1, 2])
def test_loop_ring_actions_env_and_updates(world, G):
    N, B, cap_frames, seed, T = 64, 64, 4, 9, 6
    env = make_env(world, N)
    S = sacd(batch_size=B, replay_capacity=N * cap_frames, lockstep_envs=N, seed=seed, trainers=G)
    S.init_params(4)
    ref = make_env(world, N)                              # the same scenarios, stepped with the ring's actions
    ring = R.Ring(N * cap_frames, N, G)
    X = twin(S, N, G, seed)
    for it in range(T):
        engine().sac_train_run(env, S, 1, do_update=False)
        ring.commit()
    assert S.replay_size() == ring.count == min(T, cap_frames) * N
    first = T - ring.count // N
    for k in range(ring.count // N):
        s, a, r, s2, d = S.gather(np.arange(k * N, (k + 1) * N))
        assert a.dtype == np.int32 and a.min() >= 0 and a.max() < 27
        # the act pass of iteration first + k on these observations, its Philox counter restated
        u = np.concatenate([R.u01(R.philox(R.trainer_key((seed ^ R.K_NOISE_SALT), R.K_NOISE_SALT, g), R.SAC_ACT_CTR | (first + k),
                                           np.arange(N // G))[:, 0]) for g in range(G)])
        assert np.array_equal(X.act(dev(s), u=dev(u)).cpu().numpy(), a), k
    # env outputs: a run of the discrete-27 step fed the same actions (from the start, so every frame is replayed)
    env2 = make_env(world, N)
    S2 = sacd(batch_size=B, replay_capacity=N * 16, lockstep_envs=N, seed=seed, trainers=G)
    S2.init_params(4)
    engine().sac_train_run(env2, S2, T, do_update=False)
    for k in range(T):
        s, a, r, s2, d = S2.gather(np.arange(k * N, (k + 1) * N))
        out = ref.step(dev(a))
        assert_same(out["obs"].cpu().numpy(), s2, "obs %d" % k)
        assert_same(out["reward"].cpu().numpy().astype(np.float32), r, "reward %d" % k)
        assert np.array_equal(out["done"].cpu().numpy().astype(np.uint8), d), k
    # ring-sampled updates equal update_batch on the gathered rows, bit for bit
    for _ in range(3):
        engine().sac_train_run(env, S, 1, do_update=False)
        ring.commit()
        X2 = twin(S, B, G, seed)
        sc = S.scalars()
        idx = [R.sample(seed, sc["epoch"] + 1, ring.count_g(), B, g) for g in range(G)]
        s, a, r, s2, d = S.gather(np.concatenate([ring.logical(idx[g], g) for g in range(G)]))
        l_ring, l_batch = torch.zeros(4 * G, device="cuda"), torch.zeros(4 * G, device="cuda")
        S.update_replay(losses=l_ring)
        X2.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), losses=l_batch)
        torch.cuda.synchronize()
        assert np.array_equal(l_ring.cpu().numpy(), l_batch.cpu().numpy())
        for role in range(14):
            assert np.array_equal(S.get_params(role), X2.get_params(role)), role
        assert np.array_equal(S.alpha(), X2.alpha())
        X2.close()
    st = engine().sac_train_run(env, S, 4)
    assert st.updates == 4 and np.isfinite(st.last_loss)
    ev = engine().sac_eval_run(env, S, 16, mean_action=True)
    assert ev["n_records"] + ev["unfinished"] == 16
    for x in (env, ref, env2, S, S2, X):
        x.close()


# ------------------------------------------------------------------ grouped trainers
@pytest.mark.parametrize("G", [2, 16, 32])
def test_grouped_trainers_equal_standalone(G):
    B = 64
    rng = np.random.default_rng(G)
    S = sacd(batch_size=B, seed=7, trainers=G)
    S.init_params(3)
    al = np.stack([[np.log(0.01) + 0.3 * g, 0.0, 0.0] for g in range(G)]).astype(np.float32)
    S.set_alpha(al)
    solo = []
    for g in range(G):
        X = sacd(batch_size=B, seed=7 + g)
        for role in range(11):
            X.set_params(role, S.get_params(role)[g])
        X.set_scalars(*al[g], 0, 0)
        solo.append(X)
    s = rng.normal(0, 1, (G * B, 100)).astype(np.float32); s2 = rng.normal(0, 1, (G * B, 100)).astype(np.float32)
    a = rng.integers(0, 27, G * B).astype(np.int32); r = rng.normal(0, 3, G * B).astype(np.float32)
    d = (rng.uniform(size=G * B) < 0.2).astype(np.float32)
    lg = torch.zeros(4 * G, device="cuda")
    S.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d), losses=lg)
    ls = []
    for g, X in enumerate(solo):
        l1 = torch.zeros(4, device="cuda")
        sl = slice(g * B, (g + 1) * B)
        X.update_batch(dev(s[sl]), dev(a[sl]), dev(r[sl]), dev(s2[sl]), dev(d[sl]), losses=l1)
        ls.append(l1)
    torch.cuda.synchronize()
    for role in range(14):
        allp = S.get_params(role)
        for g, X in enumerate(solo):
            assert_same(allp[g], X.get_params(role), "role %d trainer %d" % (role, g))
    for g in range(G):
        assert_same(lg.cpu().numpy()[4 * g:4 * g + 4], ls[g].cpu().numpy(), "losses %d" % g)
        assert_same(S.alpha()[g], solo[g].alpha()[0], "alpha %d" % g)
    # get_action: trainer g acts on block g with its own key
    obs = rng.normal(0, 1, (G * 8, 100)).astype(np.float32)
    ag = S.act(dev(obs)).cpu().numpy()
    for g, X in enumerate(solo):
        assert np.array_equal(ag[8 * g:8 * g + 8], X.act(dev(obs[8 * g:8 * g + 8])).cpu().numpy()), g
    # Federated_Learning_AC: every actor becomes the float32 sum, in trainer order
    actors = S.get_params(0)
    want = actors[0].copy()
    for g in range(1, G):
        want = (want + actors[g]).astype(np.float32)
    S.federate_actors()
    got = S.get_params(0)
    for g in range(G):
        assert_same(got[g], want, "federated actor %d" % g)
    for X in solo:
        X.close()
    S.close()


# ------------------------------------------------------------------ refusals
def refused(fn, text):
    with pytest.raises(Exception) as e:
        fn()
    assert text in str(e.value), str(e.value)


def test_refusals(world):
    E = engine()
    S = sacd(batch_size=64, replay_capacity=64 * 4, lockstep_envs=64)
    z = torch.zeros((64, 100), device="cuda")
    ai = torch.zeros(64, dtype=torch.int32, device="cuda")
    zr = torch.zeros(64, device="cuda")
    refused(lambda: S.per_enable(), "uavrl_sac_per_enable (prioritised replay) is not available on a discrete SAC learner")
    refused(lambda: S.update_batch_per(z, ai, zr, z, zr, zr), "uavrl_sac_update_batch_per (prioritised replay) is not available")
    refused(lambda: S.connect_self(), "uavrl_sac_comm_init is not available on a discrete SAC learner")
    refused(lambda: S.update_replay_dp(64), "uavrl_sac_update_replay_dp is not available on a discrete SAC learner")
    refused(lambda: S.critic_grads(64, batch=(z, ai, zr, z, zr)), "uavrl_sac_critic_grads_batch is not available on a discrete")
    refused(lambda: S.apply_critic_grads(), "uavrl_sac_apply_critic_grads is not available on a discrete")
    refused(lambda: S.update_batch(z, zr, zr, z, zr), "a discrete SAC learner takes int32 actions")
    env = make_env(world, 64)
    refused(lambda: E.sac_train_run_dp(env, S, 1, 64), "uavrl_sac_train_run_dp is not available on a discrete SAC learner")
    S26 = sacd(A=26, batch_size=64, replay_capacity=64 * 4, lockstep_envs=64)
    refused(lambda: E.sac_train_run(env, S26, 1), "a discrete SAC learner in the loop must have act_dim 27")
    refused(lambda: E.sac_eval_run(env, S26, 4), "a discrete SAC learner must have act_dim 27")
    for bad in (dict(A=1), dict(A=32), dict(obs=132), dict(obs=6), dict(hid=0), dict(hid=129)):
        kw = dict(obs=100, hid=64, A=27); kw.update(bad)
        with pytest.raises(Exception):
            sacd(**kw)
    big = max(E.sac_smem_bytes(128, 128, 0, 31, True))
    assert big > SMEM_MAX
    refused(lambda: sacd(128, 128, 31), "too large")
    # the continuous learner refuses the discrete act
    C = E.SacLearner(batch_size=64)
    from uavrl_b200 import _lib
    from uavrl_b200.engine import check
    refused(lambda: check(_lib.lib().uavrl_sac_act_discrete(C.h, z.data_ptr(), 64, None, 0, ai.data_ptr(), None)),
            "uavrl_sac_act_discrete needs a discrete SAC learner")
    for x in (S, S26, C, env):
        x.close()
