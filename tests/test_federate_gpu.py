"""Selective federated aggregation across grouped trainers (uavrl_learner_federate, Learner.federate,
PathPlan_City.Federated_Learning_choice :644-684) on the device.

The judge is the numpy restatement tests/fl_restatement.py, pinned to the reference's own run in test_federate_cpu.py.
Each trainer changes only in its own round, so every round is checked on its own (fl_restatement.check_rounds)."""
import os

import numpy as np
import pytest
import torch

from fl_restatement import check_rounds
from gpu_util import DEV, ROOT, city_and_params, env_dict
from shapes import SHAPES, pick
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

S = 10
# one network per route of shapes.SHAPES: tensor-core FIXED, tensor-core generic, fp32 only (in_dim % 4 != 0)
ROUTE_NETS = {"fixed": pick(100, [60], 27, 1)[:4], "generic": pick(100, [64, 32], 27, 1)[:4], "fp32": pick(99, [64], 27, 0)[:4]}
for _s in ROUTE_NETS.values():
    assert any(tuple(x[:4]) == (_s[0], _s[1], _s[2], _s[3]) for x in SHAPES), _s


@pytest.fixture(scope="module")
def fl_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "fl_golden.npz"))


def make(shape, G, seed=3, tc=True, **kw):
    in_dim, hidden, nA, dueling = shape
    kw.setdefault("replay_capacity", 64 * G)
    L = engine.Learner(in_dim, hidden, nA, bool(dueling), algo=engine.ALGO_DDQN, seed=seed, trainers=G, **kw)
    L.init_params(seed)
    _lib.lib().uavrl_learner_set_tensor_cores(L.h, int(tc))
    return L


def snapshot(L):
    return [L.get_params(w).reshape(L.G, L.P).copy() for w in range(4)], L.counters()


def run_explicit(L, probes):
    pr = torch.tensor(probes, device=DEV)
    idx, losses, chosen = L.federate(probe_states=pr, want_details=True)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), losses.cpu().numpy(), chosen.cpu().numpy()


def assert_untouched(b, a):
    (vb, cb), (va, ca) = b, a
    for w in (1, 2, 3):
        assert np.array_equal(vb[w], va[w]), "vector %d changed" % w
    assert cb == ca


# ---------------------------------------------------------------- 1. golden: the reference's own run, bit for bit
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "fp32"])
@pytest.mark.parametrize("name", ["ddqn5", "duel6"])
def test_golden_bit_for_bit(fl_golden, name, tc):
    k = lambda s: fl_golden["%s_%s" % (name, s)]             # noqa: E731
    G, dueling, hidden = int(k("G")), int(k("dueling")), [int(h) for h in k("hidden")]
    L = make((100, hidden, 27, dueling), G, tc=tc)
    L.set_params(k("local0"), 0)
    b = snapshot(L)
    idx, losses, chosen = run_explicit(L, k("probes"))
    a = snapshot(L)
    assert np.array_equal(chosen, k("chosen")), (chosen, k("chosen"))
    assert np.array_equal(a[0][0], k("local1"))
    assert_untouched(b, a)
    assert (idx == -1).all()
    L.close()


# ---------------------------------------------------------------- 2. every round at every route
LEGS = [(r, tc, G) for r in ROUTE_NETS for tc in ((True, False) if r != "fp32" else (False,)) for G in (2, 3, 8, 33, 256)]


@pytest.mark.parametrize("route,tc,G", LEGS, ids=["%s-%s-G%d" % (r, "tc" if t else "fp32", g) for r, t, g in LEGS])
def test_rounds_vs_float64(route, tc, G):
    shape = ROUTE_NETS[route]
    L = make(shape, G, seed=5 + G, tc=tc)
    rng = np.random.default_rng(G)
    probes = rng.uniform(-1, 1, size=(G, S, shape[0])).astype(np.float32)
    b = snapshot(L)
    _, losses, chosen = run_explicit(L, probes)
    a = snapshot(L)
    assert_untouched(b, a)
    check_rounds(b[0][0], a[0][0], probes, losses, chosen, shape, range(G))
    if G >= 3:
        assert not np.array_equal(a[0][0], b[0][0])
    L.close()


# ---------------------------------------------------------------- 3. weight images refreshed
@pytest.mark.parametrize("route,tc", [("fixed", True), ("generic", True), ("fixed", False)])
def test_images_refreshed(route, tc):
    shape, G = ROUTE_NETS[route], 8
    L = make(shape, G, seed=9, tc=tc)
    rng = np.random.default_rng(1)
    run_explicit(L, rng.uniform(-1, 1, size=(G, S, shape[0])).astype(np.float32))
    F = make(shape, G, seed=9, tc=tc)
    for w in range(4):
        F.set_params(L.get_params(w), w)
    F.set_counters(*L.counters())
    n = 64 * G
    obs = torch.tensor(rng.uniform(-1, 1, size=(n, shape[0])).astype(np.float32), device=DEV)
    a1, q1 = L.act(obs, 0.3, want_q=True)
    a2, q2 = F.act(obs, 0.3, want_q=True)
    assert torch.equal(a1, a2) and torch.equal(q1, q2)
    B = 32 * G
    batch = (torch.tensor(rng.uniform(-1, 1, size=(B, shape[0])).astype(np.float32), device=DEV),
             torch.tensor(rng.integers(0, shape[2], B).astype(np.int32), device=DEV),
             torch.tensor(rng.normal(size=B).astype(np.float32), device=DEV),
             torch.tensor(rng.uniform(-1, 1, size=(B, shape[0])).astype(np.float32), device=DEV),
             torch.tensor((rng.uniform(size=B) < 0.2).astype(np.float32), device=DEV))
    L.update_batch(*batch)
    F.update_batch(*batch)
    for w in range(4):
        assert np.array_equal(L.get_params(w), F.get_params(w)), w
    L.close(); F.close()


# ---------------------------------------------------------------- 4. probes from the lockstep ring
def ring_learner(env_golden, env27_golden, G, Ng, seed):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N = G * Ng
    pool = engine.EnvBatch(city, params, N, max_subgoals=64).make_scenarios(N, seed=3)
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=False)
    env.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
    env.reset(0)
    shape = (100, [64, 64], 27, 0)
    L = make(shape, G, seed=seed, replay_capacity=N * 64, lockstep_envs=N)
    engine.train_run(env, L, 30, eps=0.5)
    return L, env, shape


def test_ring_probes(env_golden, env27_golden):
    G, Ng = 4, 16
    L, env, shape = ring_learner(env_golden, env27_golden, G, Ng, 21)
    n_g = L.replay_size() // G
    assert n_g >= S
    N = G * Ng
    # a tape: echoed, and the probes are the tape's rows of each trainer's own block
    rng = np.random.default_rng(4)
    tape = np.stack([rng.choice(n_g, S, replace=False) for _ in range(G)])
    b = snapshot(L)
    idx, losses, chosen = L.federate(probe_tape=tape, want_details=True)
    a = snapshot(L)
    assert np.array_equal(idx.cpu().numpy(), tape)
    probes = np.stack([L.gather((tape[g] // Ng) * N + g * Ng + tape[g] % Ng)[0] for g in range(G)])
    check_rounds(b[0][0], a[0][0], probes, losses.cpu().numpy(), chosen.cpu().numpy(), shape, range(G))
    assert_untouched(b, a)
    # Philox draws: distinct, in range, and the same again for the same learner state and call counter
    L2, _, _ = ring_learner(env_golden, env27_golden, G, Ng, 21)
    L2.federate(probe_tape=tape)
    i1 = L.federate(want_details=True)[0].cpu().numpy()
    i2 = L2.federate(want_details=True)[0].cpu().numpy()
    assert np.array_equal(i1, i2)
    for row in i1:
        assert len(set(row.tolist())) == S and (row >= 0).all() and (row < n_g).all()
    i3 = L.federate(want_details=True)[0].cpu().numpy()
    assert not np.array_equal(i1, i3)                    # the next call draws again
    L.close(); L2.close()


# ---------------------------------------------------------------- 5. large G
def test_large_g_4096():
    G, shape = 4096, (100, [64, 64], 27, 0)
    L = make(shape, G, seed=1)
    rng = np.random.default_rng(6)
    probes = rng.uniform(-1, 1, size=(G, S, 100)).astype(np.float32)
    b = snapshot(L)
    _, losses, chosen = run_explicit(L, probes)
    a = snapshot(L)
    assert_untouched(b, a)
    rounds = sorted(rng.choice(G, 64, replace=False).tolist())
    check_rounds(b[0][0], a[0][0], probes, losses, chosen, shape, rounds)
    L.close()


# ---------------------------------------------------------------- 6. refusals
def test_refusals(env_golden, env27_golden):
    shape, G = (100, [64, 64], 27, 0), 4
    free0 = torch.cuda.mem_get_info()[0]
    L = make(shape, G, seed=2, lockstep_envs=64, replay_capacity=64 * 16)
    b = snapshot(L)
    pr = torch.zeros((G, S, 100), device=DEV)
    tape_dev = torch.zeros((G, S), dtype=torch.int32, device=DEV)
    with pytest.raises(_lib.UavrlError, match="not both"):
        L.federate(probe_states=pr, probe_tape=tape_dev)
    with pytest.raises(_lib.UavrlError, match="at least 10 transitions"):
        L.federate()                                     # empty ring
    P = make(shape, G, seed=2)                           # no lockstep ring at all
    with pytest.raises(_lib.UavrlError, match="at least 10 transitions"):
        P.federate()
    P.close()
    with pytest.raises(ValueError, match="distinct"):
        L.federate(probe_tape=np.zeros((G, S), np.int64))
    with pytest.raises(ValueError, match="lie in"):
        L.federate(probe_tape=np.tile(np.arange(S), (G, 1)) + 10 ** 6)
    torch.cuda.synchronize()
    a = snapshot(L)
    assert all(np.array_equal(x, y) for x, y in zip(b[0], a[0])) and b[1] == a[1]
    # G = 1 does nothing; G = 2 keeps every parameter
    one = make(shape, 1, seed=2)
    p1 = one.get_params(0)
    one.federate(probe_states=torch.zeros((1, S, 100), device=DEV))
    assert np.array_equal(one.get_params(0), p1)
    one.close()
    L.close()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] >= free0 - (8 << 20)


# ---------------------------------------------------------------- 7. the env plug-in
def test_env_plugin_is_fl(tmp_path):
    import importlib
    cwd = os.getcwd()
    os.chdir(ROOT)
    mod = importlib.import_module("uavrl_b200.plugins.PathPlan_City_B200")
    orig = mod.XML2Dict

    def patched(path):
        d = orig(path)
        if "Trainer" in d and isinstance(d["Trainer"], dict):
            d["Trainer"].update(Batch_Size="16", replay_size="512", save_loop="0", model_path=str(tmp_path))
        return d
    mod.XML2Dict = patched
    try:
        env = mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml", Is_FL="1", FL_Loop="2"))
        L = env.Trainer._learner
        calls, fed = [], L.federate
        L.federate = lambda *a, **k: (calls.append(env.epoch), fed(*a, **k))[1]
        for _ in range(4):
            before = L.get_params(0)
            env.run_eposide(0.3)
            changed = not np.array_equal(before, L.get_params(0))
            assert changed                                # training (and, on even episodes, aggregation) moved q_local
        assert calls == [2, 4]
        off = mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml"))
        assert off.Is_FL == 0 and off.FL_Loop == 3

        def boom(*a, **k):
            raise AssertionError("federate called with Is_FL = 0")
        off.Trainer._learner.federate = boom
        off.run_eposide(0.3)
        with pytest.raises(ValueError, match="Is_AC"):
            mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml", Is_FL="1", Is_AC="1"))
        single = mod.PathPlan_City_B200(env_dict("Trainer_DDQN_B200.xml", Is_FL="1", FL_Loop="1", num_trainers="1"))
        single.Trainer._learner.federate = boom
        single.run_eposide(0.3)                          # one trainer: accepted, nothing to aggregate
    finally:
        mod.XML2Dict = orig
        os.chdir(cwd)
