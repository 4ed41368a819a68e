"""Grouped learners (uavrl_learner_create_trainers): G independent trainers in one handle.  The defining property is checked
bit for bit: trainer g computes exactly what a stand-alone learner with its parameters, seed + g, replay_capacity / G and
lockstep_envs / G computes -- act passes, explicit updates, ring-sampled updates and the whole lockstep loop."""
import os

import numpy as np
import pytest
import torch

from gpu_util import city_and_params, env_plugin
from test_qnet_shapes_gpu import SHAPES, SHIPPED
from test_tc_gpu import big_inputs
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
G = 4


def learner(shape, trainers=1, seed=7, **kw):
    in_dim, hidden, n_actions, dueling = shape[:4]
    kw.setdefault("algo", engine.ALGO_DQN)
    kw.setdefault("batch_size", 64)
    return engine.Learner(in_dim, hidden, n_actions, dueling, seed=seed, trainers=trainers, **kw)


def standalone_like(grouped, shape, g, seed=7, **kw):
    """Trainer g of `grouped` as a stand-alone learner: its parameters and optimiser state, seed + g."""
    s = learner(shape, 1, seed + g, **kw)
    for which in range(4):
        s.set_params(grouped.get_params(which)[g], which)
    return s


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def shape_id(s):
    return "%d-%s-%d-%s" % (s[0], "x".join(map(str, s[1])), s[2], "duel" if s[3] else "q")


ACT_SHAPES = SHIPPED + [SHAPES[0][:4]]         # the four shipped networks and one generic-route shape


@pytest.mark.parametrize("shape", ACT_SHAPES, ids=shape_id)
def test_act_blocks_equal_standalone(dqn_golden, shape):
    Ng = 1000                                          # ragged last tile of every tile size
    rng = np.random.default_rng(1)
    Lg = learner(shape, G)
    Lg.init_params(3)
    assert Lg.get_params(0).shape == (G, Lg.P)
    solo = [standalone_like(Lg, shape, g) for g in range(G)]
    obs = torch.tensor(big_inputs(dqn_golden, G * Ng, rng, shape[0]), device=DEV)
    u = torch.tensor(rng.random(G * Ng).astype(np.float32), device=DEV)
    ra = torch.tensor(rng.integers(0, shape[2], G * Ng).astype(np.int32), device=DEV)
    for tc in (True, False):
        for L in [Lg] + solo:
            L.set_tensor_cores(tc)
        a, q = Lg.act(obs, 0.3, u_tape=u, rand_tape=ra, want_q=True)
        ap = Lg.act(obs, 0.3)                          # Philox draws: keyed by seed + g and the trainer-local row
        for g, S in enumerate(solo):
            blk = slice(g * Ng, (g + 1) * Ng)
            a1, q1 = S.act(obs[blk].contiguous(), 0.3, u_tape=u[blk].contiguous(), rand_tape=ra[blk].contiguous(), want_q=True)
            ap1 = S.act(obs[blk].contiguous(), 0.3)
            assert_same(q[blk].cpu().numpy(), q1.cpu().numpy(), "Q, trainer %d, tc=%s" % (g, tc))
            assert_same(a[blk].cpu().numpy(), a1.cpu().numpy(), "actions (tapes), trainer %d" % g)
            assert_same(ap[blk].cpu().numpy(), ap1.cpu().numpy(), "actions (Philox), trainer %d" % g)


def batch(dqn_golden, rng, n, shape):
    s = torch.tensor(big_inputs(dqn_golden, n, rng, shape[0]), device=DEV)
    s2 = torch.tensor(big_inputs(dqn_golden, n, rng, shape[0]), device=DEV)
    a = torch.tensor(rng.integers(0, shape[2], n).astype(np.int32), device=DEV)
    r = torch.tensor(rng.normal(0, 1, n).astype(np.float32), device=DEV)
    d = torch.tensor((rng.random(n) < 0.1).astype(np.float32), device=DEV)
    return s, a, r, s2, d


def assert_trainers_equal(Lg, solo, losses=None, solo_losses=None):
    for which, what in enumerate(("local", "target", "exp_avg", "exp_avg_sq", "grad")):
        allp = Lg.get_params(which).reshape(-1, Lg.P)
        for g, S in enumerate(solo):
            assert_same(allp[g], S.get_params(which), "%s of trainer %d" % (what, g))
    if losses is not None:
        for g in range(len(solo)):
            assert_same(losses[g:g + 1], solo_losses[g], "loss of trainer %d" % g)
    for S in solo:
        assert S.counters() == Lg.counters()


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "fp32"])
@pytest.mark.parametrize("B", [64, 6000, 9000])     # 32- / 64-row tiles, TD fused / separate (132 SMs)
@pytest.mark.parametrize("algo,shape", [(engine.ALGO_DQN, SHIPPED[0]), (engine.ALGO_DDQN, SHIPPED[0]),
                                        (engine.ALGO_DUELING, SHIPPED[2])], ids=["dqn", "ddqn", "dueling"])
def test_explicit_update_equals_standalone(dqn_golden, algo, shape, B, tc):
    rng = np.random.default_rng(B + algo)
    Lg = learner(shape, G, algo=algo, update_loop=3)
    Lg.init_params(5)
    solo = [standalone_like(Lg, shape, g, algo=algo, update_loop=3) for g in range(G)]
    for L in [Lg] + solo:
        L.set_tensor_cores(tc)
    if tc:
        assert Lg.route(B)["train_rows"] == (32 if B == 64 else 64)
    for _ in range(4):                                 # update_loop = 3: a hard update inside the window
        s, a, r, s2, d = batch(dqn_golden, rng, G * B, shape)
        loss = torch.zeros(G, device=DEV)
        Lg.update_batch(s, a, r, s2, d, loss)
        solo_loss = []
        for g, S in enumerate(solo):
            blk = slice(g * B, (g + 1) * B)
            l1 = torch.zeros(1, device=DEV)
            S.update_batch(s[blk].contiguous(), a[blk].contiguous(), r[blk].contiguous(), s2[blk].contiguous(), d[blk].contiguous(), l1)
            solo_loss.append(l1.cpu().numpy())
        assert_trainers_equal(Lg, solo, loss.cpu().numpy(), solo_loss)


def make_env(env_golden, env27_golden, n, pool):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=False)
    env.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
    return env


def test_index_tape_maps_to_ring_rows(env_golden, env27_golden):
    Ng, B, shape = 64, 64, SHIPPED[0]
    N = G * Ng
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=3)
    env = make_env(env_golden, env27_golden, N, pool)
    env.reset(0)
    Lg = learner(shape, G, algo=engine.ALGO_DDQN, replay_capacity=G * Ng * 16, lockstep_envs=N)
    Lg.init_params(2)
    engine.train_run(env, Lg, 10, eps=0.5, do_update=False)
    n_g = Lg.replay_size() // G
    assert n_g == 10 * Ng
    rng = np.random.default_rng(0)
    tape = np.stack([rng.choice(n_g, B, replace=False) for _ in range(G)]).astype(np.int32)
    solo = [standalone_like(Lg, shape, g, algo=engine.ALGO_DDQN) for g in range(G)]
    loss = torch.zeros(G, device=DEV)
    Lg.update(torch.tensor(tape, device=DEV), loss)
    solo_loss = []
    for g, S in enumerate(solo):
        k = tape[g].astype(np.int64)
        s, a, r, s2, d = Lg.gather((k // Ng) * N + g * Ng + k % Ng)
        l1 = torch.zeros(1, device=DEV)
        S.update_batch(*(torch.tensor(x, device=DEV) for x in (s, a, r, s2, d.astype(np.float32))), l1)
        solo_loss.append(l1.cpu().numpy())
    assert_trainers_equal(Lg, solo, loss.cpu().numpy(), solo_loss)


@pytest.mark.parametrize("algo", [engine.ALGO_DQN, engine.ALGO_DDQN], ids=["dqn", "ddqn"])
def test_lockstep_loop_equals_standalone_pairs(env_golden, env27_golden, algo):
    Ng, B, shape, iters = 384, 64, SHIPPED[0], 100
    N, cap_g = G * Ng, Ng * 40                          # the ring wraps within the 100 iterations
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=5)
    env = make_env(env_golden, env27_golden, N, pool)
    env.reset(0)
    Lg = learner(shape, G, seed=11, algo=algo, replay_capacity=G * cap_g, lockstep_envs=N, update_loop=3)
    Lg.init_params(1)
    st = engine.train_run(env, Lg, iters, eps=0.2)
    assert st.episodes_ended == 0 and st.env_steps == iters * N
    pairs, losses = [], []
    for g in range(G):
        e1 = make_env(env_golden, env27_golden, Ng, pool)
        e1.reset(g * Ng)
        L1 = learner(shape, 1, seed=11 + g, algo=algo, replay_capacity=cap_g, lockstep_envs=Ng, update_loop=3)
        L1.init_params(1 + g)
        s1 = engine.train_run(e1, L1, iters, eps=0.2)
        assert s1.episodes_ended == 0 and s1.updates == st.updates
        pairs.append((e1, L1)); losses.append(np.float32(s1.last_loss))
    assert_trainers_equal(Lg, [L1 for _, L1 in pairs])
    assert np.float32(st.last_loss) == np.float32(sum(float(x) for x in losses) / G)
    sg = env.get_state()
    n_g = Lg.replay_size() // G
    for g, (e1, L1) in enumerate(pairs):
        s1 = e1.get_state()
        for k in sg:
            assert_same(sg[k][g * Ng:(g + 1) * Ng], s1[k], "env state %s, block %d" % (k, g))
        assert L1.replay_size() == n_g
        k = np.arange(n_g, dtype=np.int64)
        ring_g = Lg.gather((k // Ng) * N + g * Ng + k % Ng)
        for x, y, what in zip(ring_g, L1.gather(k), ("s", "a", "r", "s2", "d")):
            assert_same(x, y, "ring %s, trainer %d" % (what, g))
    # one more ring-sampled update: every trainer's own loss slot against its pair's loss
    loss = torch.zeros(G, device=DEV)
    Lg.update(loss=loss)
    solo_loss = []
    for _, L1 in pairs:
        l1 = torch.zeros(1, device=DEV)
        L1.update(loss=l1)
        solo_loss.append(l1.cpu().numpy())
    assert_trainers_equal(Lg, [L1 for _, L1 in pairs], loss.cpu().numpy(), solo_loss)


def test_refusals_and_round_trips(dqn_golden):
    shape = SHIPPED[0]
    for bad in (0, 65536):                              # one grid row per trainer: gridDim.y <= 65535
        with pytest.raises(engine.UavrlError, match="n_trainers must be in"):
            learner(shape, bad)
    with pytest.raises(engine.UavrlError, match="multiple of n_trainers"):
        learner(shape, 3, lockstep_envs=64)
    Lg = learner(shape, G, lockstep_envs=64)
    assert Lg.trainer_count() == G
    x = torch.zeros((6, shape[0]), device=DEV)
    one = torch.zeros(6, device=DEV)
    with pytest.raises(engine.UavrlError, match="multiple of the trainer count"):
        Lg.act(x, 0.1)
    with pytest.raises(engine.UavrlError, match="multiple of the trainer count"):
        Lg.update_batch(x, one.int(), one, x, one)
    with pytest.raises(engine.UavrlError, match="uavrl_replay_push"):
        Lg.push(x, one.int(), one, x, one.to(torch.uint8))
    with pytest.raises(engine.UavrlError, match="prioritised replay"):
        Lg.per_enable()
    with pytest.raises(engine.UavrlError, match="update_batch_per"):
        Lg.update_batch_per(x[:4], one[:4].int(), one[:4], x[:4], one[:4])
    with pytest.raises(engine.UavrlError, match="comm_init"):
        Lg.connect_self()
    with pytest.raises(engine.UavrlError, match="compute_grads"):
        Lg.compute_grads(64)
    with pytest.raises(engine.UavrlError, match="apply_grads"):
        Lg.apply_grads()
    s4, a4, r4, s24, d4 = (t[:4] for t in (x, one.int(), one, x, one))
    with pytest.raises(ValueError, match="4 trainers writes 4 losses"):   # one loss per trainer: a [1] tensor would overflow
        Lg.update_batch(s4, a4, r4, s24, d4, torch.zeros(1, device=DEV))
    with pytest.raises(ValueError, match="4 trainers writes 4 losses"):
        Lg.update(loss=torch.zeros(1, device=DEV))
    # [G][P] round trip of every vector
    rng = np.random.default_rng(0)
    for which in range(5):
        p = rng.normal(0, 1, (G, Lg.P)).astype(np.float32)
        Lg.set_params(p, which)
        assert_same(Lg.get_params(which), p, "round trip %d" % which)
    # G = 1 from the new entry point is the learner uavrl_learner_create makes
    L1 = learner(shape, 1, algo=engine.ALGO_DDQN)
    L0 = learner(shape, 1, algo=engine.ALGO_DDQN)
    _lib.lib().uavrl_learner_destroy(L0.h)
    L0.h = _lib.VP()
    engine.check(_lib.lib().uavrl_learner_create(_lib.C.byref(L0.cfg), _lib.C.byref(L0.h)))
    L1.init_params(4)
    for which in (0, 1):
        L0.set_params(L1.get_params(which), which)
    s, a, r, s2, d = batch(dqn_golden, rng, 256, shape)
    for L in (L0, L1):
        L.update_batch(s, a, r, s2, d)
    assert_trainers_equal(L1, [L0])
    assert_same(L0.act(s, 0.5).cpu().numpy(), L1.act(s, 0.5).cpu().numpy(), "actions")


class CountTransfers:
    """Counts a learner's get_params / set_params calls: each moves the whole [G][P] vector between host and device."""

    def __init__(self, L):
        self.get = self.set = 0
        get, set_ = L.get_params, L.set_params

        def g(*a, **k):
            self.get += 1
            return get(*a, **k)

        def s(*a, **k):
            self.set += 1
            return set_(*a, **k)
        L.get_params, L.set_params = g, s


def env_dict(**kw):
    """The shipped env configuration with num_UAV = num_trainers = 8 and the DDQN trainer."""
    from uavrl_b200.plugins import xmlconfig
    ed = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", "PathPlan_City_B200.xml"))["simulator"]["env"]
    ed["num_UAV"], ed["scenario_pool"], ed["num_trainers"] = "8", "64", "8"
    ed["Obstacles"]["buildings"] = os.path.join(ROOT, "configs", "buildings.xml")
    ed["Agent"]["Trainer"]["Trainer_path"] = os.path.join(ROOT, "configs", "Trainer_DDQN_B200.xml")
    ed.update(kw)
    return ed


def test_env_plugin_one_trainer_per_uav(tmp_path):
    """num_UAV = num_trainers = 8: the reference's one trainer per UAV.  run_eposide runs, save() writes one q_local / q_target
    pair per trainer in the reference's per-UAV naming, and Load_Mod in a fresh env restores every trainer bit for bit.  Both
    move each of the four vectors between host and device once, whatever the trainer count."""
    with env_plugin(tmp_path) as mod:
        env = mod.PathPlan_City_B200(env_dict())
        with pytest.raises(ValueError, match="multiple of num_trainers"):
            mod.PathPlan_City_B200(env_dict(num_trainers="3"))
        with pytest.raises(ValueError, match="num_trainers = 1"):
            mod.PathPlan_City_B200(env_dict(host_driven="1"))
        tr = env.Trainer
        assert tr._learner.trainer_count() == 8 and tr.names == ["UAV_%d" % i for i in range(8)]
        info = env.run_eposide(0.3)
        assert info["updates"] > 0 and np.isfinite(info["loss"])
        n = CountTransfers(tr._learner)
        tr.save()
        assert (n.get, n.set) == (4, 0)
        env2 = mod.PathPlan_City_B200(env_dict())                   # Load_Mod in the constructor
        n = CountTransfers(env2.Trainer._learner)
        env2.Trainer.Load_Mod(str(tmp_path))
        assert (n.get, n.set) == (4, 4)
    files = sorted(os.listdir(tmp_path))
    assert files == sorted(["q_%s_DDQN_UAV_%d.pth" % (k, i) for k in ("local", "target") for i in range(8)]), files
    ck = torch.load(os.path.join(tmp_path, "q_local_DDQN_UAV_5.pth"), weights_only=False)
    assert set(ck) == {"model", "optimizer", "epoch"}
    assert_same(ck["model"]["fc1.weight"].numpy().ravel(), tr._learner.get_params(0)[5][:64 * 100], "trainer 5 fc1.weight")
    for which in range(4):
        assert_same(env2.Trainer._learner.get_params(which), tr._learner.get_params(which), "restored vector %d" % which)
    assert env2.Trainer._learner.counters() == tr._learner.counters()


def test_env_plugin_skips_malformed_checkpoints(tmp_path, capsys):
    """Of 8 trainers' checkpoint pairs, trainer 2's q_local holds a network of the wrong size and trainer 6's q_target a
    renamed key.  As in the reference (DuelingDQN_Trainer.py:56-57), the constructor prints each error and carries on: those
    two trainers keep their fresh parameters and moments, every other trainer is restored bit for bit."""
    with env_plugin(tmp_path) as mod:
        tr = mod.PathPlan_City_B200(env_dict()).Trainer                  # no files yet: fresh parameters
        fresh = [tr._rows(which) for which in range(4)]
        rng = np.random.default_rng(5)
        saved = [rng.normal(0, 1, f.shape).astype(np.float32) for f in fresh]
        for which in range(4):
            tr._learner.set_params(saved[which], which)
        tr._learner.set_counters(123, 45)
        tr.save()
        pl, pt = (os.path.join(tmp_path, "q_%s_DDQN_UAV_%d.pth" % kg) for kg in (("local", 2), ("target", 6)))
        ck = torch.load(pl, weights_only=False)
        ck["model"]["fc1.weight"] = ck["model"]["fc1.weight"][:, :99].clone()   # a network of 99 inputs
        torch.save(ck, pl)
        ck = torch.load(pt, weights_only=False)
        ck["model"] = {("fc0.bias" if k == "fc1.bias" else k): t for k, t in ck["model"].items()}
        torch.save(ck, pt)
        capsys.readouterr()
        tr2 = mod.PathPlan_City_B200(env_dict()).Trainer                 # Load_Mod in the constructor
        out = capsys.readouterr().out
    assert "q_local_DDQN_UAV_2.pth: fc1.weight is (64, 99)" in out and "q_target_DDQN_UAV_6.pth holds" in out, out
    for which in range(4):
        got = tr2._rows(which)
        for g in range(8):
            want = fresh[which][g] if g in (2, 6) else saved[which][g]
            assert_same(got[g], want, "vector %d of trainer %d" % (which, g))
    assert tr2._learner.counters() == (123, 45)
