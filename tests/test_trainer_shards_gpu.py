"""Trainer groups sharded over ranks: W learners of G / W trainers each (seeded seed + r G / W) and env shards of N / W envs
(reset stride N) compute what one learner of G trainers on the N-env batch computes, and the two aggregations
(Learner.fed_* / federate_sharded, SacLearner.fed_* / federate_actors_sharded) leave every shard where the one-GPU
federate() / federate_actors() leaves its trainers, bit for bit.

Ranks are simulated on one device: W handles, and each all-gather is a torch.cat of the handles' slices copied back into
every handle's exchange buffer."""
import numpy as np
import pytest
import torch

from fl_restatement import check_rounds
from gpu_util import DEV, SAC_ROLES, assert_same, sac, short_episode_env
from shapes import pick
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

S = 10
ROUTE_NETS = {"fixed": pick(100, [60], 27, 1)[:4], "generic": pick(100, [64, 32], 27, 1)[:4], "fp32": pick(99, [64], 27, 0)[:4]}
SHIPPED = (100, [64, 64], 27, 0)


def make(shape, G, seed, tc=True, **kw):
    in_dim, hidden, nA, dueling = shape
    kw.setdefault("replay_capacity", 64 * G)
    L = engine.Learner(in_dim, hidden, nA, bool(dueling), algo=engine.ALGO_DDQN, seed=seed, trainers=G, **kw)
    L.init_params(seed)
    L.set_tensor_cores(tc)
    return L


def shards_like(full, shape, W, seed, tc, **kw):
    """W learners holding the rows of `full`'s trainers [r G / W, (r + 1) G / W), seeded seed + r G / W."""
    GL = full.G // W
    out = []
    for r in range(W):
        L = make(shape, GL, seed + r * GL, tc, **kw)
        for w in range(4):
            L.set_params(full.get_params(w).reshape(full.G, -1)[r * GL:(r + 1) * GL], w)
        L.set_counters(*full.counters())
        L.fed_shard(r, W)
        out.append(L)
    return out


def gather(xs):
    """The all-gather of equal slices: rank r's slice of its own buffer into every buffer."""
    W = len(xs)
    full = torch.cat([x.chunk(W)[r] for r, x in enumerate(xs)])
    for x in xs:
        x.copy_(full)


def federate_sim(shards, probes=None, tape=None):
    """One sharded aggregation across the simulated ranks: (probe indices, losses and chosen lists of every rank)."""
    W, GL = len(shards), shards[0].G
    G = W * GL
    k = (G - 1) // 2
    idx = torch.empty((G, S), dtype=torch.int32, device=DEV)
    outs = [(torch.full((G, G), 7.0, device=DEV), torch.zeros((G, max(1, k)), dtype=torch.int32, device=DEV)) for _ in shards]
    for r, L in enumerate(shards):
        rows = slice(r * GL, (r + 1) * GL)
        L.fed_local(None if probes is None else probes[rows].contiguous(), None if tape is None else tape[rows].contiguous(), idx[rows])
    gather([L.fed_exchange_tensor(0) for L in shards])
    for L in shards:
        L.fed_columns()
    gather([L.fed_exchange_tensor(1) for L in shards])
    for L, (lo, ch) in zip(shards, outs):
        L.fed_rounds(lo, ch)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), [(lo.cpu().numpy(), ch.cpu().numpy()) for lo, ch in outs]


def assert_shards_equal(full, shards, what=""):
    GL = shards[0].G
    for w in range(4):
        allp = full.get_params(w).reshape(full.G, -1)
        for r, L in enumerate(shards):
            assert_same(L.get_params(w).reshape(GL, -1), allp[r * GL:(r + 1) * GL], "%s vector %d of rank %d" % (what, w, r))
    for L in shards:
        assert L.counters() == full.counters()


def assert_images_equal(full, shards, shape, rng):
    """The weight images the act pass reads (fp32 and tensor-core) hold the aggregated q_local."""
    GL, n = shards[0].G, 32
    obs = torch.tensor(rng.uniform(-1, 1, size=(full.G * n, shape[0])).astype(np.float32), device=DEV)
    _, q = full.act(obs, 0.0, want_q=True)
    for r, L in enumerate(shards):
        _, qr = L.act(obs[r * GL * n:(r + 1) * GL * n].contiguous(), 0.0, want_q=True)
        assert torch.equal(qr, q[r * GL * n:(r + 1) * GL * n]), "Q of rank %d" % r


# ---------------------------------------------------------------- 1. aggregation, explicit probes, every route
LEGS = [(rt, W, GL) for rt in ROUTE_NETS for W in (2, 3, 4) for GL in (1, 2, 5)]


@pytest.mark.parametrize("route,W,GL", LEGS, ids=["%s-W%d-GL%d" % x for x in LEGS])
def test_aggregation_explicit(route, W, GL):
    shape, G = ROUTE_NETS[route], W * GL
    tc = route != "fp32"
    full = make(shape, G, 5 + G, tc)
    shards = shards_like(full, shape, W, 5 + G, tc)
    rng = np.random.default_rng(G)
    probes = torch.tensor(rng.uniform(-1, 1, size=(G, S, shape[0])).astype(np.float32), device=DEV)
    before = full.get_params(0).reshape(G, -1).copy()
    fi, fl, fc = [t.cpu().numpy() for t in full.federate(probe_states=probes, want_details=True)]
    idx, outs = federate_sim(shards, probes=probes)
    assert (idx == -1).all() and (fi == -1).all()
    for r, (lo, ch) in enumerate(outs):
        assert_same(lo, fl, "losses of rank %d" % r)
        assert np.array_equal(ch, fc), "chosen lists of rank %d" % r
    assert_shards_equal(full, shards)
    assert_images_equal(full, shards, shape, rng)
    check_rounds(before, full.get_params(0).reshape(G, -1), probes.cpu().numpy(), fl, fc, shape, range(G))
    for L in shards + [full]:
        L.close()


def test_world_one_is_federate():
    shape, G = SHIPPED, 6
    full = make(shape, G, 3)
    (one,) = shards_like(full, shape, 1, 3, True)
    probes = torch.tensor(np.random.default_rng(0).uniform(-1, 1, size=(G, S, 100)).astype(np.float32), device=DEV)
    full.federate(probe_states=probes)
    federate_sim([one], probes=probes)
    assert_shards_equal(full, [one])
    full.close(); one.close()


# ---------------------------------------------------------------- 2. env shards
def test_env_shard_matches_full_batch_rows(env_golden, env27_golden):
    city, params = short_episode_env(env_golden, env27_golden)
    N, W, P, first = 96, 4, 331, 17
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(P, seed=3)

    def env(n):
        e = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=True)
        e.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
        return e
    full = env(N)
    full.reset(first)
    shards = []
    for r in range(W):
        e = env(N // W)
        e.set_reset_stride(N)
        e.reset(first + r * N // W)
        shards.append(e)
    rng = np.random.default_rng(1)
    restarts = 0
    for t in range(60):
        a = rng.integers(0, 27, N).astype(np.int32)
        out = full.step(torch.tensor(a, device=DEV))
        restarts += int(out["ended"].sum())
        for r, e in enumerate(shards):
            e.step(torch.tensor(a[r * N // W:(r + 1) * N // W], device=DEV))
        want = full.get_state()
        for r, e in enumerate(shards):
            got = e.get_state()
            for k, v in want.items():
                assert np.array_equal(got[k], v[r * N // W:(r + 1) * N // W]), (t, r, k)
    assert restarts >= 2 * N                             # several auto-resets per env
    with pytest.raises(_lib.UavrlError, match="stride"):
        shards[0].set_reset_stride(0)


# ---------------------------------------------------------------- 3. end to end: lockstep training, aggregation between chunks
def ring_pair(env_golden, env27_golden, W, GL, Ng, make_learner):
    city, params = short_episode_env(env_golden, env27_golden)
    G = W * GL
    N = G * Ng
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(3 * N, seed=7)

    def env(n, first, stride):
        e = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=True)
        e.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
        e.set_reset_stride(stride)
        e.reset(first)
        return e
    full = (env(N, 5, N), make_learner(G, N, 0))
    shards = [(env(N // W, 5 + r * N // W, N), make_learner(GL, N // W, r * GL)) for r in range(W)]
    return full, shards


E2E = [("tc", True, False), ("tc-per", True, True), ("fp32", False, False), ("fp32-per", False, True)]


@pytest.mark.parametrize("W,GL", [(2, 2), (4, 1)], ids=["W2-GL2", "W4-GL1"])
@pytest.mark.parametrize("name,tc,per", E2E, ids=[e[0] for e in E2E])
def test_train_run_sharded_equals_one_gpu(env_golden, env27_golden, name, tc, per, W, GL):
    Ng, cap = 32, 32 * 20

    def mk(G, n, first):
        L = make(SHIPPED, G, 11 + first, tc, replay_capacity=cap * G, lockstep_envs=n, batch_size=32)
        L.init_params(11 + first)
        if per:
            L.per_enable_trainers()
        return L
    (fe, fl), shards = ring_pair(env_golden, env27_golden, W, GL, Ng, mk)
    for r, (_, L) in enumerate(shards):
        L.fed_shard(r, W)
    for chunk in range(3):
        fs = engine.train_run(fe, fl, 16, 0.4)
        ss = [engine.train_run(e, L, 16, 0.4) for e, L in shards]
        assert fs.episodes_ended == sum(s.episodes_ended for s in ss)
        assert fs.env_steps == sum(s.env_steps for s in ss)
        fi, flo, fc = [t.cpu().numpy() for t in fl.federate(want_details=True)]
        idx, outs = federate_sim([L for _, L in shards])
        assert np.array_equal(idx, fi), chunk
        for lo, ch in outs:
            assert_same(lo, flo, "losses")
            assert np.array_equal(ch, fc)
        assert_shards_equal(fl, [L for _, L in shards], "chunk %d" % chunk)
    n_slots = (cap // Ng + 1) * Ng
    if per:
        leaves, totals, beta = fl.per_state(n_slots)
        leaves, totals = leaves.reshape(W * GL, -1), np.asarray(totals).reshape(-1)
        for r, (_, L) in enumerate(shards):
            l2, t2, b2 = L.per_state(n_slots)
            assert_same(np.asarray(l2).reshape(GL, -1), leaves[r * GL:(r + 1) * GL], "leaves of rank %d" % r)
            assert_same(np.asarray(t2).reshape(-1), totals[r * GL:(r + 1) * GL], "totals of rank %d" % r)
            assert b2 == beta
    # the rings: trainer g's k-th oldest transition (logical (k / Ng) N + g Ng + k % Ng of the full ring)
    N, NL = W * GL * Ng, GL * Ng
    k = np.arange(0, fl.replay_size() // (W * GL), 7)
    for r, (_, L) in enumerate(shards):
        for j in range(GL):
            g = r * GL + j
            want = fl.gather((k // Ng) * N + g * Ng + k % Ng)
            got = L.gather((k // Ng) * NL + j * Ng + k % Ng)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (r, j)
    for _, L in shards + [(fe, fl)]:
        L.close()


@pytest.mark.parametrize("per", [False, True], ids=["uniform", "per"])
def test_sac_train_run_sharded_equals_one_gpu(env_golden, env27_golden, per):
    W, GL, Ng, cap = 2, 2, 32, 32 * 20

    def mk(G, n, first):
        S_ = sac(G, 7 + first, replay_capacity=cap * G, lockstep_envs=n, batch_size=32)
        S_.init_params(7 + first)
        if per:
            S_.per_enable()
        return S_
    (fe, fs), shards = ring_pair(env_golden, env27_golden, W, GL, Ng, mk)
    for r, (_, X) in enumerate(shards):
        X.fed_shard(r, W)
    for chunk in range(3):
        engine.sac_train_run(fe, fs, 16)
        for e, X in shards:
            engine.sac_train_run(e, X, 16)
        fs.federate_actors()
        sac_federate_sim([X for _, X in shards])
        assert_sac_shards_equal(fs, [X for _, X in shards])
    if per:
        n = fs.tree_slots()
        leaves, totals, beta = fs.per_state(n)
        for r, (_, X) in enumerate(shards):
            l2, t2, b2 = X.per_state(n)
            assert_same(np.asarray(l2), np.asarray(leaves)[r * GL:(r + 1) * GL], "leaves of rank %d" % r)
            assert b2 == beta
    for _, X in shards + [(fe, fs)]:
        X.close()


# ---------------------------------------------------------------- 4. SAC actor aggregation
def sac_federate_sim(shards):
    for X in shards:
        X.fed_local()
    gather([X.fed_exchange_tensor() for X in shards])
    for X in shards:
        X.fed_sum_actors()
    torch.cuda.synchronize()


def assert_sac_shards_equal(full, shards):
    GL = shards[0].G
    for role in range(SAC_ROLES):
        allp = full.get_params(role).reshape(full.G, -1)
        for r, X in enumerate(shards):
            assert_same(X.get_params(role).reshape(GL, -1), allp[r * GL:(r + 1) * GL], "role %d of rank %d" % (role, r))
    al = full.alpha()
    for r, X in enumerate(shards):
        assert_same(X.alpha(), al[r * GL:(r + 1) * GL], "alpha of rank %d" % r)


@pytest.mark.parametrize("W,GL", [(W, GL) for W in (2, 3, 4) for GL in (1, 2, 5)])
def test_sac_aggregation(W, GL):
    G = W * GL
    full = sac(G, 3)
    full.init_params(3)
    shards = []
    for r in range(W):
        X = sac(GL, 3 + r * GL)
        for role in range(11):
            X.set_params(role, full.get_params(role).reshape(G, -1)[r * GL:(r + 1) * GL])
        X.set_alpha(full.alpha()[r * GL:(r + 1) * GL])
        X.fed_shard(r, W)
        shards.append(X)
    full.federate_actors()
    sac_federate_sim(shards)
    assert_sac_shards_equal(full, shards)
    obs = torch.tensor(np.random.default_rng(2).uniform(-1, 1, size=(G * 8, 100)).astype(np.float32), device=DEV)
    eps = torch.zeros((G * 8, 2), device=DEV)
    a = full.act(obs, eps)
    for r, X in enumerate(shards):                      # the actor images
        rows = slice(r * GL * 8, (r + 1) * GL * 8)
        assert torch.equal(X.act(obs[rows].contiguous(), eps[rows].contiguous()), a[rows])
    for X in shards + [full]:
        X.close()


# ---------------------------------------------------------------- 5. refusals leave the handle untouched
def snapshot(L):
    return [L.get_params(w).copy() for w in range(4)], L.counters()


def assert_untouched(L, b):
    a = snapshot(L)
    for w in range(4):
        assert np.array_equal(a[0][w], b[0][w])
    assert a[1] == b[1]


def test_refusals(env_golden, env27_golden):
    L = make(SHIPPED, 2, 1, lockstep_envs=32, replay_capacity=32 * 16)
    b = snapshot(L)
    st = L.fed_local
    with pytest.raises(_lib.UavrlError, match="before uavrl_learner_fed_shard"):
        st(torch.zeros((2, S, 100), device=DEV))
    with pytest.raises(_lib.UavrlError, match="before uavrl_learner_fed_shard"):
        L.fed_columns()
    with pytest.raises(ValueError, match="fed_shard"):
        L.fed_exchange_tensor(0)
    for rank, world in ((-1, 2), (2, 2), (0, 0)):
        with pytest.raises(_lib.UavrlError, match="rank in"):
            L.fed_shard(rank, world)
    with pytest.raises(_lib.UavrlError, match="65535"):
        L.fed_shard(0, 32768)
    L.fed_shard(1, 2)
    with pytest.raises(_lib.UavrlError, match="out of order"):
        L.fed_columns()
    with pytest.raises(_lib.UavrlError, match="out of order"):
        L.fed_rounds()
    with pytest.raises(_lib.UavrlError, match="at least 10 transitions"):
        L.fed_local()                                    # empty ring
    with pytest.raises(_lib.UavrlError, match="not both"):
        L.fed_local(torch.zeros((2, S, 100), device=DEV), torch.zeros((2, S), dtype=torch.int32, device=DEV))
    L.fed_local(torch.zeros((2, S, 100), device=DEV))
    with pytest.raises(_lib.UavrlError, match="out of order"):
        L.fed_rounds()
    torch.cuda.synchronize()
    assert_untouched(L, b)
    L.close()
    X = sac(2, 1)
    with pytest.raises(_lib.UavrlError, match="before uavrl_sac_fed_shard"):
        X.fed_local()
    with pytest.raises(_lib.UavrlError, match="before uavrl_sac_fed_shard"):
        X.fed_sum_actors()
    with pytest.raises(_lib.UavrlError, match="rank in"):
        X.fed_shard(3, 2)
    with pytest.raises(_lib.UavrlError, match="65535"):
        X.fed_shard(0, 40000)
    X.fed_shard(0, 2)
    with pytest.raises(_lib.UavrlError, match="out of order"):
        X.fed_sum_actors()
    X.close()
