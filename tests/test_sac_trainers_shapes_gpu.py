"""Grouped SAC trainers (uavrl_sac_create_trainers) at every shape of the SAC shape sweep, away from the shipped G = 4.  The
four SAC tile kernels launch a separate instance for one trainer, with the trainer offset compiled out, so the shape sweep
never runs the grouped instances; here G = 3 runs them at every row of shapes.SAC_SHAPES.  Trainer g must equal,
bit for bit, a stand-alone SacLearner with its parameters, moments and alpha triple, seed + g, replay_capacity / G and
Ng = lockstep_envs / G envs, and the last trainer (the largest offsets) is held to the float64 update of
sac_restatement with the SAC sweep's bounds.  The ring loop runs at one env per trainer and at G = 4096, and the actor
aggregation at every shape."""
import numpy as np
import pytest
import torch

from fl_restatement import federate_actors
from gpu_util import DEV, SAC_ROLES, assert_same, dev, distinct_alphas, ring_env, sac, sac_standalone_like, short_episode_env
from sac_restatement import A, actor_fwd, check_step, clean_batch, draw_batch, init_state, read_state, sac_update64, unpack
from shapes import SAC_SHAPES, sac_shape_id
from uavrl_b200 import engine

pytestmark = pytest.mark.gpu
G = 3
KEYS = ("actor", "c1", "c2", "t1", "t2", "actor_m", "c1_m", "c2_m", "actor_v", "c1_v", "c2_v")


class Trainer:
    """Trainer g of a grouped SacLearner, seen through the calls read_state and check_step make on a learner."""

    def __init__(self, S, g):
        self.S, self.g = S, g

    def get_params(self, role):
        return self.S.get_params(role)[self.g]

    def grads(self, role):
        return self.S.get_params(11 + role)[self.g]

    def scalars(self):
        la, m, v = (float(x) for x in self.S.alpha()[self.g])
        sc = self.S.scalars()
        return dict(log_alpha=la, la_m=m, la_v=v, epoch=sc["epoch"], adam_step=sc["adam_step"])


def grouped(shape, rng, **kw):
    """G trainers of `shape`, each from its own init_state draw, with distinct alpha triples, and their stand-alone twins."""
    obs, hid, bound, _ = shape
    net = dict(obs_dim=obs, hidden=hid, action_bound=bound)
    S = sac(G, **net, **kw)
    states = [init_state(rng, obs, hid) for _ in range(G)]
    for role, k in enumerate(KEYS):
        S.set_params(role, np.stack([st[k] for st in states]))
    distinct_alphas(S, rng)
    return S, [sac_standalone_like(S, g, **net, **kw) for g in range(G)], states


def assert_trainer_equal(S, g, X, roles=None):
    roles = roles if roles is not None else [S.get_params(r) for r in range(SAC_ROLES)]
    for role in range(SAC_ROLES):
        assert_same(roles[role][g], X.get_params(role), "role %d of trainer %d" % (role, g))
    assert_same(S.alpha()[g], X.alpha()[0], "alpha triple of trainer %d" % g)
    sg, sx = S.scalars(), X.scalars()
    assert (sg["epoch"], sg["adam_step"]) == (sx["epoch"], sx["adam_step"])


# ------------------------------------------------------------------ act
@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
def test_act_equals_standalone_and_float64(shape):
    """n = 1, 33 and 1000 rows per trainer, injected noise and Philox draws: every trainer bit for bit as its stand-alone
    learner; the last trainer's actions (injected noise) within test_sac_shapes_gpu.test_act_vs_float64's bound of float64,
    after its rows near a ReLU kink of its actor are drawn again."""
    obs, hid, bound, _ = shape
    rng = np.random.default_rng([obs, hid, 3])
    S, solo, states = grouped(shape, rng)
    P = unpack(states[G - 1]["actor"], "actor", obs, hid)
    for n in (1, 33, 1000):
        s = rng.normal(0, 1, (G * n, obs)).astype(np.float32)
        eps = rng.normal(size=(G * n, A)).astype(np.float32)
        last = slice((G - 1) * n, G * n)
        for _ in range(30):
            f = actor_fwd(P, s[last].astype(np.float64), eps[last].astype(np.float64), bound)
            near = (np.abs(f["z"]) <= 5e-5 * f["zabs"]).any(1)
            if not near.any():
                break
            s[last][near] = rng.normal(0, 1, (int(near.sum()), obs))
        assert not near.any()
        s_d, e_d = dev(s), dev(eps)
        a_inj = S.act(s_d, e_d).cpu().numpy()
        a_phi = S.act(s_d).cpu().numpy()
        for g, X in enumerate(solo):
            blk = slice(g * n, (g + 1) * n)
            assert_same(a_inj[blk], X.act(s_d[blk].contiguous(), e_d[blk].contiguous()).cpu().numpy(), ("eps", n, g))
            assert_same(a_phi[blk], X.act(s_d[blk].contiguous()).cpu().numpy(), ("Philox", n, g))
        (_, _), (Wm, bm), (Ws, bs) = P
        scale = f["h"] @ np.abs(Wm).T + np.abs(bm) + (f["h"] @ np.abs(Ws).T + np.abs(bs)) * np.abs(eps[last])
        err = np.abs(a_inj[last].astype(np.float64) - f["act"]) - bound * (1e-6 + 2e-5 * scale)
        assert (err <= 0).all(), (n, float(err.max()))
    S.close()
    for X in solo:
        X.close()


# ------------------------------------------------------------------ explicit updates
LEGS = {"B1": (1, 0), "B64": (64, 0), "B200": (200, 0), "B200-3ctas": (200, 3)}   # B per trainer, UAVRL_SAC_MAX_CTAS


@pytest.mark.parametrize("leg", list(LEGS))
@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
def test_update_equals_standalone_and_float64(shape, leg, monkeypatch):
    """4 updates: every trainer bit for bit as its stand-alone learner after each (the fourth draws its noise with Philox);
    the last trainer's first three against the float64 update (sac_restatement.check_step), its batch drawn clear of
    the float64 update's decision points."""
    obs, hid, bound, _ = shape
    B, ctas = LEGS[leg]
    if ctas:
        monkeypatch.setenv("UAVRL_SAC_MAX_CTAS", str(ctas))                 # several tiles per CTA, per trainer
    rng = np.random.default_rng([obs, hid, B, ctas])
    S, solo, _ = grouped(shape, rng, batch_size=B)
    view = Trainer(S, G - 1)
    losses = torch.zeros(4 * G, device=DEV)
    for step in range(4):
        prev = read_state(view)
        blocks = [list(draw_batch(rng, B, obs, bound)) for _ in range(G - 1)] + [clean_batch(rng, prev, B, obs, hid, bound)]
        s, a, r, s2, d, e1, e2 = (dev(np.concatenate(p)) for p in zip(*blocks))
        philox = step == 3
        if philox:
            e1 = e2 = None
        S.update_batch(s, a, r, s2, d, e1, e2, losses)
        got = losses.cpu().numpy()
        for g, X in enumerate(solo):
            blk = slice(g * B, (g + 1) * B)
            part = lambda t: None if t is None else t[blk].contiguous()  # noqa: E731
            l1 = torch.zeros(4, device=DEV)
            X.update_batch(part(s), part(a), part(r), part(s2), part(d), part(e1), part(e2), l1)
            assert_same(got[4 * g:4 * g + 4], l1.cpu().numpy(), "losses of trainer %d, step %d" % (g, step))
        roles = [S.get_params(r) for r in range(SAC_ROLES)]
        for g, X in enumerate(solo):
            assert_trainer_equal(S, g, X, roles)
        if not philox:
            new, out = sac_update64(prev, *blocks[G - 1], obs, hid, bound)
            check_step(view, prev, new, out, got[4 * (G - 1):].astype(np.float64), (leg, step))
    assert S.scalars()["epoch"] == 4 and S.scalars()["adam_step"] == 4
    S.close()
    for X in solo:
        X.close()


# ------------------------------------------------------------------ the lockstep ring
def sac_loop_pairs(env_golden, env27_golden, shape, G_, Ng, iters, frames, batch, trainers, pool_n=None, seed=11):
    """A grouped SAC learner on G_ Ng auto-resetting envs and stand-alone pairs for `trainers`, all run through `iters`
    lockstep iterations (the pool rule of test_trainers_shapes_gpu.LoopRun keeps the pairs' restarts in step); every
    trainer of `trainers` is then compared with its pair (roles, alpha, counters, env block, ring rows) and one more
    ring-sampled update's loss slots with its pair's."""
    obs, hid, bound, _ = shape
    N = G_ * Ng
    pool_n = pool_n or Ng
    assert ((G_ - 1) * Ng) % pool_n == 0
    city, params = short_episode_env(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, pool_n, max_subgoals=64).make_scenarios(pool_n, seed=5)
    net = dict(obs_dim=obs, hidden=hid, action_bound=bound, batch_size=batch)
    env = ring_env(city, params, N, pool, 0)
    S = sac(G_, seed=seed, replay_capacity=G_ * frames * Ng, lockstep_envs=N, **net)
    S.init_params(1)
    distinct_alphas(S, np.random.default_rng(seed))
    pairs = {g: (ring_env(city, params, Ng, pool, g * Ng),
                 sac_standalone_like(S, g, seed=seed, replay_capacity=frames * Ng, lockstep_envs=Ng, **net)) for g in trainers}
    st = engine.sac_train_run(env, S, iters)
    assert st.updates > 0 and st.env_steps == iters * N
    stats = {g: engine.sac_train_run(e1, X, iters) for g, (e1, X) in pairs.items()}
    assert all(s1.updates == st.updates for s1 in stats.values())
    if len(pairs) == G_:
        assert np.float32(st.last_loss) == np.float32(sum(float(np.float32(s1.last_loss)) for s1 in stats.values()) / G_)
    roles = [S.get_params(r) for r in range(SAC_ROLES)]
    sg = env.get_state()
    n_g = S.replay_size() // G_
    for g, (e1, X) in pairs.items():
        assert_trainer_equal(S, g, X, roles)
        s1 = e1.get_state()
        for k in sg:
            assert_same(sg[k][g * Ng:(g + 1) * Ng], s1[k], "env state %s, block %d" % (k, g))
        assert X.replay_size() == n_g
        k = np.arange(n_g, dtype=np.int64)
        for x, y, what in zip(S.gather((k // Ng) * N + g * Ng + k % Ng), X.gather(k), ("s", "a", "r", "s2", "d")):
            assert_same(x, y, "ring %s, trainer %d" % (what, g))
    del roles
    out = torch.zeros(4 * G_, device=DEV)
    S.update_replay(losses=out)
    out = out.cpu().numpy()
    for g, (_, X) in pairs.items():
        l1 = torch.zeros(4, device=DEV)
        X.update_replay(losses=l1)
        assert_same(out[4 * g:4 * g + 4], l1.cpu().numpy(), "losses of trainer %d after the ring update" % g)
    actors = S.get_params(0)
    for g, (_, X) in pairs.items():
        assert_same(actors[g], X.get_params(0), "actor of trainer %d after the ring update" % g)
    for e1, X in pairs.values():
        e1.close(); X.close()
    env.close(); S.close()
    return st, n_g


RING_LEGS = [(sh, Ng) for sh in SAC_SHAPES if sh[0] == 100 for Ng in (1, 37)]


@pytest.mark.parametrize("shape,Ng", RING_LEGS, ids=["%s-Ng%d" % (sac_shape_id(sh), Ng) for sh, Ng in RING_LEGS])
def test_lockstep_loop_equals_standalone_pairs(env_golden, env27_golden, shape, Ng):
    """G = 3 at the obs-100 shapes, 40 iterations through a 24-frame ring (it wraps) with episodes ending."""
    st, n_g = sac_loop_pairs(env_golden, env27_golden, shape, G, Ng, 40, 24, 16, range(G))
    assert st.episodes_ended > 0 and n_g == 24 * Ng


def test_lockstep_loop_g4096_one_env_per_trainer(env_golden, env27_golden):
    """4096 trainers of one env each at the shipped shape, batch 64, 72 iterations (updates from the 65th): trainers 0, 1,
    2047, 4094, 4095 and three drawn at random against stand-alone pairs."""
    Gb = 4096
    pick = sorted({0, 1, 2047, 4094, 4095} | set(np.random.default_rng(3).choice(Gb, 3, replace=False).tolist()))
    st, n_g = sac_loop_pairs(env_golden, env27_golden, SAC_SHAPES[0], Gb, 1, 72, 80, 64, pick, pool_n=Gb - 1)
    assert st.updates == 72 - 64 and n_g == 72


# ------------------------------------------------------------------ Federated_Learning_AC
@pytest.mark.parametrize("shape", SAC_SHAPES, ids=sac_shape_id)
def test_federate_actors_every_shape(shape):
    """Every actor becomes the float32 left-to-right sum of the G actors (full mantissas, so the order shows), nothing else
    changes, and the next act pass (Philox noise) equals stand-alone learners loaded with the summed actor: the actor
    images were refreshed."""
    obs, hid, bound, _ = shape
    rng = np.random.default_rng([obs, hid, 9])
    S = sac(G, obs_dim=obs, hidden=hid, action_bound=bound)
    before = {}
    for role in range(11):
        before[role] = rng.normal(0, 0.1, (G, S.P[role] if role < 5 else S.P[(role - 5) % 3])).astype(np.float32)
        if role >= 8:
            before[role] = np.abs(before[role])
        S.set_params(role, before[role])
    al = distinct_alphas(S, rng)
    S.federate_actors()
    torch.cuda.synchronize()
    want = federate_actors(before[0])
    assert_same(S.get_params(0), want, "every actor is the left-to-right sum")
    for role in range(1, 11):
        assert_same(S.get_params(role), before[role], "role %d untouched" % role)
    assert_same(S.alpha(), al, "alpha untouched")
    n = 33
    s = dev(rng.normal(0, 1, (G * n, obs)).astype(np.float32))
    acts = S.act(s).cpu().numpy()
    for g in range(G):
        X = sac(1, 7 + g, obs_dim=obs, hidden=hid, action_bound=bound)
        X.set_params(0, want[g])
        assert_same(acts[g * n:(g + 1) * n], X.act(s[g * n:(g + 1) * n].contiguous()).cpu().numpy(), "act after federate, %d" % g)
        X.close()
    S.close()
