"""SAC (continuous) learner beyond the shipped network (obs 100, hidden 64, action_bound 1) against a float64 restatement of
one SAC_Trainer.update (Trainer/SAC_Trainer.py:122-147, 325-379; BaseClass/BaseCNN.py:459-500): losses, the reduced gradients
of all three networks and every piece of state after each step, at batches of one tile, of ragged tiles, of several tiles
per CTA and of the benchmark's size.  Also: get_action against float64 and the Philox noise it draws, the lockstep replay ring
read back and replayed through the CPU oracle, a ring-sampled update against the same rows given explicitly, two live
learners of different shapes, and the shapes the learner refuses.  The float64 reference is sac_restatement.py,
pinned in test_sac_f64_cpu.py."""
import numpy as np
import pytest
import torch

import oracle as O
from gpu_util import dev, n_sm  # noqa: F401  (module fixture)
from sac_restatement import HP, A, actor_fwd, check_step, clean_batch, draw_batch, init_state, read_state, sac_update64, unpack
from shapes import SAC_SHAPES, sac_shape_id

gpu = pytest.mark.gpu
SMEM_LIMIT = 227 * 1024                     # shared memory one block may use


# ------------------------------------------------------------------ shapes
REFUSED = [                     # (obs_dim, hidden, message)
    (98, 64, "obs_dim must be a multiple of 4"),
    (128, 64, "obs_dim must be at most 124"),
    (100, 72, "networks too large for the SMEM-resident SAC kernels"),
    (8, 128, "networks too large for the SMEM-resident SAC kernels"),
]


def make_learner(engine, obs, hid, bound, B, st, **kw):
    S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, **HP, **kw)
    load_state(S, st)
    return S


def load_state(S, st):
    for role, k in enumerate(("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v")):
        S.set_params(role, st[k])
    S.set_scalars(st["log_alpha"], st["la_m"], st["la_v"], epoch=st["step"], adam_step=st["step"])


@pytest.fixture(scope="module")
def engine():
    from uavrl_b200 import engine as e
    return e


@gpu
def test_shape_table(engine):
    """Every row of SAC_SHAPES is accepted and fits the 227 KB a block may use; every row of REFUSED is refused with its message,
    before anything is allocated on the device."""
    for obs, hid, bound, ok in SAC_SHAPES:
        smem = engine.sac_smem_bytes(obs, hid)
        assert ok and max(smem) <= SMEM_LIMIT, (obs, hid, smem)
        S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound)
        assert S.smem_bytes() == smem
        assert S.P[0] == hid * obs + hid + 2 * (A * hid + A) and S.P[1] == hid * (obs + A) + hid + hid * hid + hid + A * hid + A
        S.close()
    assert any(h > 64 for _, h, _, _ in SAC_SHAPES) and any(h % 4 for _, h, _, _ in SAC_SHAPES) and any(h % 2 for _, h, _, _ in SAC_SHAPES)
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
        for sh in SAC_SHAPES:
            if only is None or sh[:3] in only:
                yield pytest.param(sh, leg, id="%s-%s" % (sac_shape_id(sh), leg))


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
@pytest.mark.parametrize("shape", [SAC_SHAPES[0], SAC_SHAPES[4], SAC_SHAPES[7]], ids=sac_shape_id)
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
@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
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

