"""Data-parallel SAC (include/uavrl.h, uavrl_sac_comm_init .. uavrl_sac_train_run_dp) on one GPU.

world = 1: the fused update (connect_self + update_replay_dp) and the split form without a collective equal update_replay bit
for bit, update after update, through both halves of the receive buffer and on the accumulating multi-tile path.  W = 2, 3, 4
ranks simulated in one process: each rank samples its own ring with its own seed, the test sums the ranks' exchange vectors
in float32 in rank order; every replica ends bit-identical and the step matches the float64 SAC update on the concatenated
batch (sac_restatement.sac_update64, check_step's bounds) and one update_batch on those rows.  The data-parallel loop at
world = 1 equals sac_train_run over 150 iterations.  Every refusal leaves the learner as it was."""
import numpy as np
import pytest
import torch

import replay_restatement as R
from gpu_util import SAC_ROLES, assert_same, dev, short_episode_env
from sac_restatement import HP, check_step, near_decision, read_state, sac_update64
from shapes import SAC_SHAPES, sac_shape_id
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu

RING_SHAPES = [sh for sh in SAC_SHAPES if sh[0] == 100]        # a ring holds the env's 100-float observations


@pytest.fixture(scope="module")
def city_params(env_golden, env27_golden):
    return short_episode_env(env_golden, env27_golden)


def make_pair(city_params, obs, hid, bound, B, N, cap_frames, seed, scen_seed, **kw):
    """An auto-resetting env of N UAVs (episodes end within MAX_STEP steps) and a SAC learner whose ring it fills."""
    city, params = city_params
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(256, seed=scen_seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    S = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, replay_capacity=N * cap_frames, lockstep_envs=N,
                          seed=seed, **HP, **kw)
    S.init_params(4)
    return env, S


def snapshot(S):
    """Everything an update may change: every role, the alpha triples, the scalars and the ring's size."""
    return [S.get_params(r) for r in range(SAC_ROLES)], S.alpha(), S.scalars(), S.replay_size()


def assert_replicas(S, X, what, losses=None, x_losses=None):
    """Bit-identical networks, targets, moments, alpha triple, counters (and losses); the reduced gradients as values (an
    exchange stores 0 + g, which turns -0 into +0)."""
    for r in range(SAC_ROLES):
        a, b = S.get_params(r), X.get_params(r)
        if r >= 11:
            assert np.array_equal(a, b), (what, r)
        else:
            assert_same(a, b, (what, r))
    assert_same(S.alpha(), X.alpha(), (what, "alpha"))
    assert S.scalars() == X.scalars(), what
    if losses is not None:
        assert_same(losses.cpu().numpy(), x_losses.cpu().numpy(), (what, "losses"))


def split_update(S, global_batch, batch=None, idx_tape=None, eps_next=None, eps_cur=None, losses=None):
    """The split form on one rank with no collective: the exchange vectors are the sums already."""
    S.critic_grads(global_batch, batch=batch, idx_tape=idx_tape, eps_next=eps_next)
    S.apply_critic_grads()
    S.actor_grads(eps_cur)
    S.apply_actor_grads(losses)


# ------------------------------------------------------------------ world = 1, bit for bit
@pytest.mark.parametrize("ctas", [0, 3], ids=["one-tile-per-cta", "3ctas"])
@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
def test_world1_bit_for_bit(city_params, shape, ctas, monkeypatch):
    """Six updates (both parities of the exchange tag) of batch 200 (7 tiles, the last ragged; with 3 CTAs the partials
    accumulate over tiles) with the same index and noise tapes: update_replay, the split form and connect_self +
    update_replay_dp hold the same bits after each.  A ring holds 100-float observations, so shapes with another obs_dim
    compare update_batch with the split form's explicit-batch phase."""
    obs, hid, bound, _ = shape
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))
    B, N, cap_frames = 200, 96, 4
    rng = np.random.default_rng(hid + 7 * ctas)
    if obs == 100:
        pairs = [make_pair(city_params, obs, hid, bound, B, N, cap_frames, 9, 5) for _ in range(3)]
        for env, S in pairs:
            engine.sac_train_run(env, S, 6, do_update=False)
        (_, A), (_, Sp), (_, F) = pairs
        F.connect_self()
    else:
        A, Sp = (engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=B, seed=9, **HP) for _ in range(2))
        for S in (A, Sp):
            S.init_params(4)
        F = None
    for S in (Sp, F) if F else (Sp,):
        assert_replicas(A, S, "start")
    for step in range(6):
        e1 = dev(rng.normal(size=(B, 2)).astype(np.float32)); e2 = dev(rng.normal(size=(B, 2)).astype(np.float32))
        la, ls, lf = (torch.zeros(4, device="cuda") for _ in range(3))
        if F:
            tape = dev(rng.choice(A.replay_size(), B, replace=False).astype(np.int32))
            A.update_replay(tape, e1, e2, la)
            split_update(Sp, B, idx_tape=tape, eps_next=e1, eps_cur=e2, losses=ls)
            F.update_replay_dp(B, tape, e1, e2, lf)
        else:
            rows = [dev(x) for x in (rng.normal(0, 1, (B, obs)), rng.uniform(-bound, bound, (B, 2)), rng.normal(0, 1, B),
                                     rng.normal(0, 1, (B, obs)), (rng.uniform(size=B) < 0.2))]
            rows = [x.float() for x in rows]
            A.update_batch(*rows, e1, e2, la)
            split_update(Sp, B, batch=rows, eps_next=e1, eps_cur=e2, losses=ls)
        torch.cuda.synchronize()
        assert_replicas(A, Sp, ("split", step), la, ls)
        if F:
            assert_replicas(A, F, ("fused", step), la, lf)
    assert A.scalars()["adam_step"] == 6
    if F:
        for env, S in pairs:
            env.close(); S.close()
    else:
        A.close(); Sp.close()


# ------------------------------------------------------------------ W ranks in one process
def check_or_exempt(S, prev, new, out, losses, what):
    """check_step's bounds; a batch with a row at a ReLU kink or a q1 / q2 tie of the float64 step may miss them (a sampled
    row cannot be drawn again).  Returns 1 when checked, 0 when exempt."""
    try:
        check_step(S, prev, new, out, losses, what)
        return 1
    except AssertionError:
        near, near_actor = near_decision(out)
        if not (near.any() or near_actor.any()):
            raise
        return 0


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("shape", RING_SHAPES, ids=sac_shape_id)
def test_simulated_ranks(city_params, shape, W):
    """W ranks, each with its own 64-env shard, ring and seed, run two split updates of 64 rows each; the test all-reduces the
    two exchange vectors in float32 in rank order.  Replicas stay bit-identical, and each step matches the float64 update on
    the concatenated batch (rows restated per rank seed, noise tapes concatenated), as does one update_batch on those rows."""
    obs, hid, bound, _ = shape
    B, N, cap_frames = 64, 64, 4
    ranks = [make_pair(city_params, obs, hid, bound, B, N, cap_frames, 11 + w, 20 + w) for w in range(W)]
    for env, S in ranks:
        engine.sac_train_run(env, S, 6, do_update=False)
    Ls = [S for _, S in ranks]
    ring = R.Ring(N * cap_frames, N)
    for _ in range(6):
        ring.commit()
    checked = 0
    for step in range(2):
        prev = read_state(Ls[0])
        sc = Ls[0].scalars()
        X = engine.SacLearner(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=W * B, seed=1, **HP)
        for role in range(11):
            X.set_params(role, Ls[0].get_params(role))
        X.set_scalars(sc["log_alpha"], sc["la_m"], sc["la_v"], sc["epoch"], sc["adam_step"])
        losses = [torch.zeros(4, device="cuda") for _ in range(W)]
        for S in Ls:
            S.critic_grads(W * B)
        for phase in (0, 1):
            if phase:
                for S in Ls:
                    S.actor_grads()
            xs = [S.exchange_tensor(phase) for S in Ls]
            tot = xs[0].clone()
            for x in xs[1:]:
                tot += x
            for x in xs:
                x.copy_(tot)
            for S, loss in zip(Ls, losses):
                S.apply_critic_grads() if phase == 0 else S.apply_actor_grads(loss)
        torch.cuda.synchronize()
        for S, loss in zip(Ls[1:], losses[1:]):
            assert_replicas(Ls[0], S, ("replica", step), losses[0], loss)
        epoch = sc["epoch"] + 1
        c_next, c_cur = R.sac_update_ctrs(epoch)
        parts = [Ls[w].gather(R.sample(11 + w, epoch, ring.count, B)) for w in range(W)]
        s, a, r, s2, d = (np.concatenate([p[k] for p in parts]) for k in range(5))
        e1 = np.concatenate([R.sac_noise(11 + w, c_next, B) for w in range(W)])
        e2 = np.concatenate([R.sac_noise(11 + w, c_cur, B) for w in range(W)])
        new, out = sac_update64(prev, s, a, r, s2, d.astype(np.float64), e1, e2, obs, hid, bound)
        got = losses[0].cpu().numpy().astype(np.float64)
        checked += check_or_exempt(Ls[0], prev, new, out, got, ("dp", W, step))
        lx = torch.zeros(4, device="cuda")
        X.update_batch(dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.float32)), dev(e1.astype(np.float32)),
                       dev(e2.astype(np.float32)), lx)
        torch.cuda.synchronize()
        checked += check_or_exempt(X, prev, new, out, lx.cpu().numpy().astype(np.float64), ("update_batch", W, step))
        X.close()
    assert checked >= 2
    for env, S in ranks:
        env.close(); S.close()


# ------------------------------------------------------------------ the loop
def test_loop_world1_matches_sac_train_run(city_params):
    """sac_train_run_dp after connect_self equals sac_train_run over 150 iterations (a ring of 8 frames wraps many times and
    episodes end every few steps): every role, alpha triple, counter and the envs' state, bit for bit."""
    B, N, cap_frames = 64, 64, 8
    (ep, P), (ed, D) = (make_pair(city_params, 100, 64, 1.0, B, N, cap_frames, 9, 3) for _ in range(2))
    D.connect_self()
    for env, S in ((ep, P), (ed, D)):
        engine.sac_train_run(env, S, 3, do_update=False)
    st = engine.sac_train_run(ep, P, 150)
    engine.sac_train_run_dp(ed, D, 150, B)
    torch.cuda.synchronize()
    assert st.updates == 150 and st.episodes_ended > 0
    assert_replicas(P, D, "loop")
    assert P.scalars()["epoch"] == 150 and P.replay_size() == D.replay_size() == N * cap_frames
    sp, sd = ep.get_state(), ed.get_state()
    for k in sp:
        assert_same(sp[k], sd[k], k)
    ep.close(); P.close(); ed.close(); D.close()


# ------------------------------------------------------------------ refusals
def refused(S, call, match, code=engine.UavrlError):
    """call() raises with `match`, and every role, the alpha triples, the counters and the ring are what they were."""
    before = snapshot(S)
    with pytest.raises(code, match=match):
        call()
    torch.cuda.synchronize()
    after = snapshot(S)
    for r in range(SAC_ROLES):
        assert_same(before[0][r], after[0][r], (match, r))
    assert_same(before[1], after[1], (match, "alpha"))
    assert before[2:] == after[2:], match


def test_refusals_leave_state_untouched(city_params):
    B, N = 64, 64
    env, S = make_pair(city_params, 100, 64, 1.0, B, N, 4, 9, 3)
    rows = [torch.zeros((B, 100), device="cuda"), torch.zeros((B, 2), device="cuda"), torch.zeros(B, device="cuda"),
            torch.zeros((B, 100), device="cuda"), torch.zeros(B, device="cuda")]
    # a ring that holds (the loop: would hold at its first update) <= batch_size transitions: 64 after one iteration
    refused(S, lambda: engine.sac_train_run_dp(env, S, 1, B), "before uavrl_sac_comm_connect")
    S.connect_self()
    refused(S, lambda: engine.sac_train_run_dp(env, S, 1, B), "replay holds <= batch_size")
    engine.sac_train_run(env, S, 1, do_update=False)
    refused(S, lambda: S.critic_grads(B), "replay holds <= batch_size")
    refused(S, lambda: S.update_replay_dp(B), "replay holds <= batch_size")
    engine.sac_train_run(env, S, 2, do_update=False)
    # global_batch <= 0
    for gb in (0, -B):
        refused(S, lambda: S.critic_grads(gb), "global_batch must be > 0")
        refused(S, lambda: S.critic_grads(gb, batch=rows), "global_batch must be > 0")
        refused(S, lambda: S.update_replay_dp(gb), "global_batch must be > 0")
        refused(S, lambda: engine.sac_train_run_dp(env, S, 1, gb), "bad argument")
    # phases out of order
    refused(S, S.apply_critic_grads, "out of order")
    refused(S, S.actor_grads, "out of order")
    refused(S, S.apply_actor_grads, "out of order")
    S.critic_grads(B)
    refused(S, lambda: S.critic_grads(B), "waits for its next phase")
    refused(S, lambda: S.update_replay_dp(B), "waits for its next phase")
    refused(S, S.actor_grads, "out of order")
    refused(S, S.apply_actor_grads, "out of order")
    S.apply_critic_grads()
    refused(S, S.apply_critic_grads, "out of order")
    refused(S, S.apply_actor_grads, "out of order")
    S.actor_grads()
    refused(S, S.actor_grads, "out of order")
    S.apply_actor_grads()
    S.update_replay_dp(B)                                          # back in order: the fused update runs
    env.close(); S.close()
    # no ring
    X = engine.SacLearner(batch_size=B, seed=9, **HP)
    X.connect_self()
    refused(X, lambda: X.critic_grads(B), "no replay ring")
    refused(X, lambda: X.update_replay_dp(B), "no replay ring")
    X.close()
    # not connected, with a warm ring
    env, S = make_pair(city_params, 100, 64, 1.0, B, N, 4, 9, 3)
    engine.sac_train_run(env, S, 3, do_update=False)
    refused(S, lambda: S.update_replay_dp(B), "before uavrl_sac_comm_connect")
    refused(S, lambda: engine.sac_train_run_dp(env, S, 1, B), "before uavrl_sac_comm_connect")
    env.close(); S.close()
    # several trainers
    G = engine.SacLearner(batch_size=B, seed=9, trainers=2, replay_capacity=4 * N, lockstep_envs=N, **HP)
    refused(G, lambda: G.connect_self(), "several trainers|2 trainers")
    refused(G, lambda: G.critic_grads(B), "2 trainers")
    refused(G, lambda: G.critic_grads(B, batch=rows), "2 trainers")
    refused(G, lambda: G.update_replay_dp(B), "2 trainers")
    refused(G, G.apply_critic_grads, "2 trainers")
    G.close()
