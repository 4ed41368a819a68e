"""Discrete SAC on the GPU away from init_state (SacLearner(discrete=True), include/uavrl.h "SAC, discrete actions"): the
update against the float64 restatement across policy sharpness, temperature, hyper-parameters, large |Q| and rewards and
mid-training Adam states (sac_discrete_restatement.regime_rows), on the accumulating tile path and for grouped trainers in
regimes of their own; the categorical draw's ties, rounding fallback, one-hot rows, row counts, counter and frequencies; the
lockstep loop and the policy evaluation at several shapes, bit for bit against the calls they are built from."""
import numpy as np
import pytest
import torch
from scipy import stats

import replay_restatement as R
from gpu_util import assert_records_equal, assert_same, city_and_params, compose, dev, sac, short_episode_env
from sac_discrete_restatement import (HP, WIDEST, categorical_pick, check_step, f32, fc3, init_state, mlp_fwd,
                                      pick_margin, read_state, regime_batch, regime_rows, regime_seed, regime_state, sacd_update64,
                                      set_state, sharpen, softmax, unpack)
from uavrl_b200 import _lib, engine as E

pytestmark = pytest.mark.gpu
SMEM_MAX = 232448
EVAL_NOISE_TAG = 1 << 62                 # eval.cu kEvalNoiseTag: the sampled evaluation's counters


def sacd(obs=100, hid=64, A=27, hp=HP, **kw):
    kw.setdefault("batch_size", 64)
    return E.SacLearner(obs_dim=obs, hidden=hid, act_dim=A, discrete=True, **hp, **kw)


def widest_hidden(obs, A):
    best = 0
    for h in range(1, 129):
        if max(E.sac_smem_bytes(obs, h, 0, A, True)) <= SMEM_MAX:
            best = h
    return best


def test_widest_table():
    """the restatement's WIDEST table is what the kernels fit"""
    for (A, obs), hid in WIDEST.items():
        assert widest_hidden(obs, A) == hid, (A, obs)


def run_updates(S, sts, shape, hp, bk, rng, what, steps=4):
    """`steps` updates of S (G = len(sts) trainers, B rows each) on regime batches; each trainer's update is checked entry by
    entry against its float64 step from the state S held before it.  Returns the batches."""
    A, hid, obs, B = shape
    G = len(sts)
    losses = torch.zeros(4 * G, device="cuda")
    done = []
    for step in range(steps):
        per = [regime_batch(rng, st, B, obs, hid, A, **bk) for st in sts]
        batch = [np.concatenate([p[i] for p in per]) for i in range(5)]
        S.update_batch(*(dev(x) for x in batch), losses=losses)
        torch.cuda.synchronize()
        got = losses.cpu().numpy().astype(np.float64)
        for g, st in enumerate(sts):
            new, out = sacd_update64(st, *per[g], obs, hid, A, hp)
            check_step(S, new, out, got[4 * g:4 * g + 4], (what, g, step), hp, g=None if G == 1 else g)
        sts = [read_state(S, None if G == 1 else g) for g in range(G)]
        done.append((batch, got))
    return done


# ------------------------------------------------------------------ the update in every regime
ROWS = regime_rows(WIDEST[31, 128])


@pytest.mark.parametrize("rid,shape,sk,bk,hp", ROWS, ids=[r[0] for r in ROWS])
def test_update_regimes(rid, shape, sk, bk, hp):
    A, hid, obs, B = shape
    rng = np.random.default_rng(regime_seed(rid))
    S = sacd(obs, hid, A, hp, batch_size=B)
    st = regime_state(rng, obs, hid, A, hp=hp, **sk)
    set_state(S, st)
    run_updates(S, [st], shape, hp, bk, rng, rid)
    S.close()


CORNERS = [((2, 1, 4, 33), dict(gap=120.0, alpha=50.0)), ((31, WIDEST[31, 128], 128, 4096), dict(gap=18.4, alpha=5.0, t0=1000))]


@pytest.mark.parametrize("max_ctas", [1, 2])
@pytest.mark.parametrize("G", [1, 3])
@pytest.mark.parametrize("corner", [0, 1])
def test_update_accumulates_tiles(monkeypatch, max_ctas, G, corner):
    """UAVRL_SAC_MAX_CTAS = 1 or 2: every CTA loops over several tiles and accumulates its partial (iter > 0), per trainer."""
    monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(max_ctas))
    shape, sk = CORNERS[corner]
    A, hid, obs, B = shape
    rng = np.random.default_rng(100 * max_ctas + 10 * G + corner)
    S = sacd(obs, hid, A, batch_size=B, trainers=G)
    sts = [regime_state(rng, obs, hid, A, **dict(sk, alpha=sk["alpha"] * (g + 1))) for g in range(G)]
    set_state(S, sts)
    run_updates(S, sts, shape, HP, {}, rng, ("max_ctas", max_ctas, G, corner))
    S.close()


@pytest.mark.parametrize("G,B", [(3, 1), (3, 33), (5, 1), (5, 33)])
def test_grouped_trainers_own_regimes(G, B):
    """Trainer g in a regime of its own (sharpness, alpha, Adam moments at one shared step): each against its own float64
    step, and the whole group bit for bit against stand-alone learners fed the same rows."""
    A, hid, obs = 27, 64, 100
    rng = np.random.default_rng(G * 100 + B)
    gaps, alphas = (None, 18.4, 95.0, 120.0, 40.0), (0.01, 5.0, 50.0, 0.5, 5.0)
    sts = [regime_state(rng, obs, hid, A, gap=gaps[g], alpha=alphas[g], t0=1000) for g in range(G)]
    S = sacd(batch_size=B, trainers=G, seed=7)
    set_state(S, sts)
    solo = []
    for g in range(G):
        X = sacd(batch_size=B, seed=7 + g)
        set_state(X, sts[g])
        solo.append(X)
    for step in range(4):
        cur = sts if step == 0 else [read_state(S, g) for g in range(G)]
        ((s, a, r, s2, d), lg), = run_updates(S, cur, (A, hid, obs, B), HP, {}, rng, ("grouped", G, B, step), steps=1)
        for g, X in enumerate(solo):
            sl = slice(g * B, (g + 1) * B)
            l1 = torch.zeros(4, device="cuda")
            X.update_batch(dev(s[sl]), dev(a[sl]), dev(r[sl]), dev(s2[sl]), dev(d[sl]), losses=l1)
            assert_same(lg[4 * g:4 * g + 4].astype(np.float32), l1.cpu().numpy(), "losses %d step %d" % (g, step))
        for role in range(14):
            allp = S.get_params(role)
            for g, X in enumerate(solo):
                assert_same(allp[g], X.get_params(role), "role %d trainer %d step %d" % (role, g, step))
        for g, X in enumerate(solo):
            assert_same(S.alpha()[g], X.alpha()[0], "alpha %d step %d" % (g, step))
    for X in solo + [S]:
        X.close()


# ------------------------------------------------------------------ the categorical draw
def fixed_policy(S, obs, hid, A, bias, G=1):
    """fc3's weights zero and its bias `bias` (one row per trainer): every row's probabilities are softmax(bias) whatever
    the observation"""
    rng = np.random.default_rng(3)
    bias = np.atleast_2d(np.asarray(bias, np.float64))
    acts = []
    for g in range(G):
        st = init_state(rng, obs, hid, A)
        W, b = fc3(obs, hid, A)
        st["actor"][W] = 0.0
        st["actor"][b] = f32(bias[g % bias.shape[0]])
        acts.append(st["actor"].astype(np.float32))
    S.set_params(0, acts[0] if G == 1 else np.stack(acts))


def device_probs(bias):
    """the act kernel's fp32 softmax of one row (exact when every exp is 1 or 0 and the sum an integer)"""
    b = np.asarray(bias, np.float32)
    e = np.exp(b - b.max()).astype(np.float32)
    s = np.float32(0)
    for x in e:
        s = np.float32(s + x)
    return (e / s).astype(np.float32)


def act_into(S, obs, n, u=None, mean=False, pad=64):
    """uavrl_sac_act_discrete into a buffer of n + pad sentinels: (the n actions, the pad left as written)"""
    buf = torch.full((n + pad,), -7, dtype=torch.int32, device="cuda")
    E.check(_lib.lib().uavrl_sac_act_discrete(S.h, obs.data_ptr(), n, None if u is None else u.data_ptr(), int(mean), buf.data_ptr(), None))
    out = buf.cpu().numpy()
    return out[:n], out[n:]


@pytest.mark.parametrize("A", [2, 27, 31])
def test_argmax_ties_take_the_lowest_index(A):
    S = sacd(A=A)
    x = dev(np.random.default_rng(A).normal(0, 1, (64, 100)).astype(np.float32))
    fixed_policy(S, 100, 64, A, np.zeros(A))
    assert (S.act(x, mean=True).cpu().numpy() == 0).all()
    if A > 2:
        bias = np.full(A, -1.0)
        bias[[5, A - 3]] = 0.5                          # two equal maxima, neither at index 0
        fixed_policy(S, 100, 64, A, bias)
        assert (S.act(x, mean=True).cpu().numpy() == 5).all()
    S.close()


def test_rounding_fallback_and_leading_zeros():
    """fc3 biases in {0, -200}: the fp32 probabilities are exactly 1/k or 0.  With u = 1 on the tape no cumulative sum
    exceeds u sum(p): the draw falls back to the last k with p_k > 0; u = nextafter(1, 0) reaches it through the walk, and
    u = 0 with leading zeros takes the first positive entry."""
    A, n = 27, 64
    S = sacd(A=A)
    x = dev(np.zeros((n, 100), np.float32))
    rng = np.random.default_rng(11)
    for trial in range(6):
        bias = np.where(rng.uniform(size=A) < 0.5, 0.0, -200.0)
        bias[:3] = -200.0                                # leading zeros
        bias[-4:] = -200.0                               # trailing zeros
        bias[3 + trial] = 0.0
        p = device_probs(bias)
        assert set(np.unique(p)) <= {np.float32(0), np.float32(1) / np.float32((bias == 0).sum())}
        last, first = int(np.nonzero(p)[0][-1]), int(np.nonzero(p)[0][0])
        fixed_policy(S, 100, 64, A, bias)
        one = np.float32(1.0)
        s = np.float32(0)
        for v in p:
            s = np.float32(s + v)
        assert not np.float32(one * s) < s               # u = 1: no cumulative sum exceeds u sum(p), only the fallback answers
        for u, want in ((one, last), (np.nextafter(one, np.float32(0)), last), (np.float32(0), first)):
            assert categorical_pick(p, u, np.float32) == want
            a, pad = act_into(S, x, n, u=dev(np.full(n, u, np.float32)))
            assert (a == want).all() and (pad == -7).all(), (trial, u, want, a[:4])
    S.close()


def test_one_hot_rows():
    """a bias gap of 120: fp32 p is exactly one-hot, so every u of the tape and argmax return the hot index"""
    A, n = 31, 256
    S = sacd(A=A)
    x = dev(np.random.default_rng(1).normal(0, 1, (n, 100)).astype(np.float32))
    u = np.concatenate([[0.0, 0.5, np.nextafter(np.float32(1), np.float32(0)), 1.0], np.random.default_rng(2).uniform(size=n - 4)])
    for hot in (0, 13, A - 1):
        bias = np.full(A, -120.0)
        bias[hot] = 0.0
        assert (device_probs(bias) == np.eye(A, dtype=np.float32)[hot]).all()
        fixed_policy(S, 100, 64, A, bias)
        assert (S.act(x, u=dev(u.astype(np.float32))).cpu().numpy() == hot).all()
        assert (S.act(x).cpu().numpy() == hot).all()
        assert (S.act(x, mean=True).cpu().numpy() == hot).all()
    S.close()


@pytest.mark.parametrize("n,G", [(1, 1), (31, 1), (33, 1), (4097, 1), (99, 3)])
def test_act_row_counts(n, G):
    """Every row against categorical_pick on the float64 probabilities (away from a cumulative boundary), argmax likewise, and
    no row at or past n written; trainer g draws on its own key for its block."""
    A, obs, hid = 27, 100, 64
    rng = np.random.default_rng(n + G)
    S = sacd(obs, hid, A, trainers=G, seed=21)
    sts = [sharpen(init_state(rng, obs, hid, A), rng, obs, hid, A, 6.0 + 3 * g) for g in range(G)]
    S.set_params(0, sts[0]["actor"].astype(np.float32) if G == 1 else np.stack([st["actor"].astype(np.float32) for st in sts]))
    x = rng.normal(0, 1, (n, obs)).astype(np.float32)
    ng = n // G
    p = np.concatenate([softmax(mlp_fwd(unpack(sts[g]["actor"], obs, hid, A), x[g * ng:(g + 1) * ng].astype(np.float64))["out"])
                        for g in range(G)])
    u = rng.uniform(size=n).astype(np.float32)
    for call, tape in ((0, True), (1, False)):
        if not tape:
            u = np.concatenate([R.u01(R.philox(R.trainer_key(21 ^ R.K_NOISE_SALT, R.K_NOISE_SALT, g), R.SAC_ACT_CTR | call,
                                               np.arange(ng))[:, 0]) for g in range(G)])
        a, pad = act_into(S, dev(x), n, u=dev(u) if tape else None)
        assert (pad == -7).all() and a.min() >= 0 and a.max() < A
        ok = np.array([pick_margin(p[i], u[i]) > 1e-5 for i in range(n)])
        want = np.array([categorical_pick(p[i], u[i]) for i in range(n)])
        assert ok.mean() > 0.9 and np.array_equal(a[ok], want[ok]), (call, tape)
    m, pad = act_into(S, dev(x), n, mean=True)
    srt = np.sort(p, 1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-5 * srt[:, -1]
    assert (pad == -7).all() and np.array_equal(m[clear], p.argmax(1)[clear])
    S.close()


def test_act_counter():
    """mean=True draws nothing and leaves the act counter; a tape call advances it as a Philox call does"""
    A, obs, hid, n, seed = 27, 100, 64, 512, 5
    rng = np.random.default_rng(4)
    S = sacd(obs, hid, A, seed=seed)
    st = sharpen(init_state(rng, obs, hid, A), rng, obs, hid, A, 5.0)
    S.set_params(0, st["actor"].astype(np.float32))
    x = rng.normal(0, 1, (n, obs)).astype(np.float32)
    p = softmax(mlp_fwd(unpack(st["actor"], obs, hid, A), x.astype(np.float64))["out"])

    def philox_call(call):
        uu = R.u01(R.philox(R.trainer_key(seed ^ R.K_NOISE_SALT, R.K_NOISE_SALT, 0), R.SAC_ACT_CTR | call, np.arange(n))[:, 0])
        ok = np.array([pick_margin(p[i], uu[i]) > 1e-5 for i in range(n)])
        return ok, np.array([categorical_pick(p[i], uu[i]) for i in range(n)])
    S.act(dev(x), mean=True)
    ok, want = philox_call(0)
    a = S.act(dev(x)).cpu().numpy()                      # call 0: the mean call before it counted nothing
    assert np.array_equal(a[ok], want[ok])
    S.act(dev(x), u=dev(rng.uniform(size=n).astype(np.float32)))       # call 1, on the tape
    S.act(dev(x), mean=True)
    ok, want = philox_call(2)
    a = S.act(dev(x)).cpu().numpy()
    assert np.array_equal(a[ok], want[ok])
    S.close()


@pytest.mark.parametrize("A", [2, 31])
def test_act_frequencies_chi_square_grouped(A):
    """2^20 draws per trainer of G = 2 at fixed probabilities of their own"""
    G, n = 2, 1 << 20
    rng = np.random.default_rng(A)
    S = sacd(A=A, trainers=G, seed=99)
    ps = [rng.dirichlet(np.ones(A) * 2.0) for _ in range(G)]
    fixed_policy(S, 100, 64, A, np.log(np.stack(ps)), G)
    a = S.act(torch.zeros((G * n, 100), device="cuda")).cpu().numpy()
    for g in range(G):
        p = device_probs(np.log(ps[g])).astype(np.float64)
        counts = np.bincount(a[g * n:(g + 1) * n], minlength=A)
        assert counts.size == A
        chi2 = ((counts - n * p) ** 2 / (n * p)).sum()
        assert stats.chi2.sf(chi2, A - 1) > 1e-4, (g, chi2)
    S.close()


# ------------------------------------------------------------------ the lockstep loop
@pytest.fixture(scope="module")
def world(env_golden, env27_golden):
    return city_and_params(env_golden, env27_golden)[:2]


def make_env(world, N, seed=8):
    city, params = world
    env = E.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(1024, seed=seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    return env


def twin(S, hid, B, G, seed):
    X = sacd(hid=hid, batch_size=B, seed=seed, trainers=G)
    for role in range(11):
        X.set_params(role, S.get_params(role))
    sc = S.scalars()
    X.set_scalars(sc["log_alpha"], sc["la_m"], sc["la_v"], sc["epoch"], sc["adam_step"])
    X.set_alpha(S.alpha())
    return X


@pytest.mark.parametrize("hid,N,G,B,cap", [(1, 96, 3, 1, 3), (32, 256, 4, 33, 5), (WIDEST[27, 100], 96, 1, 256, 3),
                                           (WIDEST[27, 100], 256, 4, 256, 5), (32, 96, 4, 33, 3)])
def test_loop_shapes(world, hid, N, G, B, cap):
    """The ring's actions are the act pass on the restated Philox tape, after the ring has wrapped; every ring-sampled update
    equals update_batch on the gathered rows, bit for bit."""
    seed, T = 9, cap + 3
    env = make_env(world, N)
    S = sacd(hid=hid, batch_size=B, replay_capacity=N * cap, lockstep_envs=N, seed=seed, trainers=G)
    S.init_params(4)
    ring = R.Ring(N * cap, N, G)
    X = twin(S, hid, N, G, seed)
    for it in range(T):
        E.sac_train_run(env, S, 1, do_update=False)
        ring.commit()
    assert S.replay_size() == ring.count == cap * N
    first = T - ring.count // N
    for k in range(ring.count // N):
        s, a, r, s2, d = S.gather(np.arange(k * N, (k + 1) * N))
        u = np.concatenate([R.u01(R.philox(R.trainer_key(seed ^ R.K_NOISE_SALT, R.K_NOISE_SALT, g), R.SAC_ACT_CTR | (first + k),
                                           np.arange(N // G))[:, 0]) for g in range(G)])
        assert np.array_equal(X.act(dev(s), u=dev(u)).cpu().numpy(), a), k
    for _ in range(3):
        E.sac_train_run(env, S, 1, do_update=False)
        ring.commit()
        X2 = twin(S, hid, B, G, seed)
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
    for x in (env, S, X):
        x.close()


# ------------------------------------------------------------------ policy evaluation
def eval_env(env_golden, env27_golden, N, P, auto_reset):
    city, params = short_episode_env(env_golden, env27_golden)
    env = E.EnvBatch(city, params, N, max_subgoals=64, auto_reset=auto_reset)
    sc = env.make_scenarios(P, seed=5)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    return env


def learner_snapshot(S):
    return [S.get_params(r) for r in range(11)] + [S.alpha(), np.array([S.scalars()[k] for k in ("epoch", "adam_step")])]


def eval_counter(first, it):
    return EVAL_NOISE_TAG | (first << 31) | it


@pytest.mark.parametrize("mean", [True, False], ids=["argmax", "sampled"])
@pytest.mark.parametrize("G", [1, 4])
def test_discrete_eval_equals_composition(env_golden, env27_golden, G, mean):
    """sac_eval_run with a discrete learner: the records equal the suite driven through act and the discrete-27 step --
    argmax p, or draws on the restated tape (trainer g's key, counter kEvalNoiseTag | first << 31 | iteration, one row per
    env) -- and the learner's parameters and act counter are as before."""
    N, P, n, first, seed = 64, 200, 96, 3, 13
    S = sacd(trainers=G, seed=seed)
    S.init_params(4)
    rng = np.random.default_rng(G)
    sts = [read_state(S, None if G == 1 else g) for g in range(G)]
    for g, st in enumerate(sts):
        sharpen(st, rng, 100, 64, 27, 4.0 + g)
    S.set_params(0, sts[0]["actor"].astype(np.float32) if G == 1 else np.stack([st["actor"].astype(np.float32) for st in sts]))
    before = learner_snapshot(S)
    E1 = eval_env(env_golden, env27_golden, N, P, False)
    res = E.sac_eval_run(E1, S, n, first_scenario=first, mean_action=mean)
    assert res["unfinished"] == 0
    for a, b in zip(before, learner_snapshot(S)):
        assert_same(a, b, "learner after the evaluation")
    X = twin(S, 64, 64, G, seed)
    it = [0]

    def act(o):
        if mean:
            return X.act(o, mean=True), _lib.ACT_DISCRETE27
        u = np.concatenate([R.u01(R.philox(R.trainer_key(seed ^ R.K_NOISE_SALT, R.K_NOISE_SALT, g), eval_counter(first, it[0]),
                                           np.arange(N // G))[:, 0]) for g in range(G)])
        it[0] += 1
        return X.act(o, u=dev(u)), _lib.ACT_DISCRETE27
    E2 = eval_env(env_golden, env27_golden, N, P, True)
    assert_records_equal(res["records"], compose(E2, n, first, act), ("discrete", G, mean))
    # the act counter: S's next Philox draw is still call 0
    x = np.random.default_rng(5).normal(0, 1, (N, 100)).astype(np.float32)
    u = np.concatenate([R.u01(R.philox(R.trainer_key(seed ^ R.K_NOISE_SALT, R.K_NOISE_SALT, g), R.SAC_ACT_CTR | 0,
                                       np.arange(N // G))[:, 0]) for g in range(G)])
    assert np.array_equal(S.act(dev(x)).cpu().numpy(), X.act(dev(x), u=dev(u)).cpu().numpy())
    for h in (S, X, E1, E2):
        h.close()


@pytest.mark.parametrize("G", [1, 4])
def test_continuous_sampled_eval_equals_composition(env_golden, env27_golden, G):
    """sac_eval_run's sampled continuous actions on the restated noise (sac_noise on trainer g's key and the evaluation's
    counters).  The host's Box-Muller differs from the kernel's by a few ulp, so the composition's actions may differ in the
    last bit: integer fields must agree, lengths and scores to 1e-4 relative."""
    N, P, n, first, seed = 64, 200, 96, 5, 17
    S = sac(trainers=G, seed=seed)
    S.init_params(6)
    before = learner_snapshot(S)
    E1 = eval_env(env_golden, env27_golden, N, P, False)
    res = E.sac_eval_run(E1, S, n, first_scenario=first)
    assert res["unfinished"] == 0
    for a, b in zip(before, learner_snapshot(S)):
        assert_same(a, b, "learner after the evaluation")
    it = [0]

    def act(o):
        eps = np.concatenate([R.sac_noise(seed, eval_counter(first, it[0]), N // G, g) for g in range(G)]).astype(np.float32)
        it[0] += 1
        return S.act(o, eps=dev(eps)), _lib.ACT_CONT_F32X2
    E2 = eval_env(env_golden, env27_golden, N, P, True)
    want = compose(E2, n, first, act)
    got = res["records"]
    for k in E.RECORD_FIELDS:
        if np.issubdtype(np.asarray(want[k]).dtype, np.floating):
            np.testing.assert_allclose(got[k], want[k], rtol=1e-4, atol=1e-4, err_msg=k)
        else:
            assert np.array_equal(got[k], want[k]), k
    for h in (S, E1, E2):
        h.close()
