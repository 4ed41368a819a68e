"""Shared helpers for the -m gpu parity tests (CUDA path vs the CPU oracle / golden vectors): device tensors, the env
fixtures, the env plug-in configuration, and the grouped-trainer helpers that build a trainer's stand-alone twin and compare
the two bit for bit."""
import contextlib
import importlib
import os

import numpy as np
import pytest
import torch

import oracle as O
import uavrl_b200  # noqa: F401
from sac_restatement import HP
from uavrl_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
PER_MAX = 4194304                      # n1 = 131 072 group sums, n2 = 4096 = kPerMaxL2: the sampler's whole prefix scan
MAX_STEP = 12                          # short_episode_env: episodes end within the loops, so done transitions enter the rings
SAC_ROLES = 14                         # 0-4 networks, 5-10 Adam moments, 11-13 last gradients


def dev(x, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(x)).cuda()
    return t if dt is None else t.to(dt)


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def city_and_params(env_golden, env27_golden):
    g = env_golden
    city = engine.City(g["dims"][0], g["dims"][1], g["dims"][2], g["buildings"])
    p = g["uav_params"]
    params = engine.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    ocity = O.OracleCity(g["dims"][0], g["dims"][1], g["dims"][2], g["buildings"])
    oparams = O.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    return city, params, ocity, oparams


def assert_close64(a, b, tol=1e-9, what=""):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    err = np.abs(a - b) / np.maximum(1.0, np.abs(b))
    assert err.max() <= tol, (what, float(err.max()), int(err.argmax()))


BIN = np.r_[11:86, 90:95]          # the 80 occupancy probes: exact {0,1}
REAL = np.r_[0:11, 86:90, 95:100]  # real-valued entries


def assert_obs(got, want64, what=""):
    """got: fp32 obs from the GPU; want64: fp64 obs of the oracle/reference.  North-star tolerance:
    1e-5 on real-valued entries, occupancy bits exact."""
    got = np.asarray(got); want64 = np.asarray(want64, np.float64)
    assert np.array_equal(got[..., BIN], want64[..., BIN].astype(np.float32)), what
    np.testing.assert_allclose(got[..., REAL], want64[..., REAL], rtol=1e-5, atol=1e-5, err_msg=what)


@contextlib.contextmanager
def env_plugin(model_path, **trainer):
    """The env plug-in module, run from the repository root, whose trainers read a small batch and replay, no periodic
    save and checkpoints under model_path; `trainer` overrides further Trainer XML entries (strings)."""
    cwd = os.getcwd()
    os.chdir(ROOT)
    mod = importlib.import_module("uavrl_b200.plugins.PathPlan_City_B200")
    orig = mod.XML2Dict

    def patched(path):
        d = orig(path)
        if "Trainer" in d and isinstance(d["Trainer"], dict):
            d["Trainer"].update({**dict(Batch_Size="16", replay_size="512", save_loop="0", model_path=str(model_path)), **trainer})
        return d
    mod.XML2Dict = patched
    try:
        yield mod
    finally:
        mod.XML2Dict = orig
        os.chdir(cwd)


def env_dict(trainer, agent=None, **kw):
    """The shipped env configuration with num_UAV = num_trainers = 8, the Trainer XML `trainer` and, when given, the Agent
    XML `agent` (file names under configs/)."""
    from uavrl_b200.plugins import xmlconfig
    ed = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", "PathPlan_City_B200.xml"))["simulator"]["env"]
    ed["num_UAV"], ed["scenario_pool"], ed["num_trainers"] = "8", "64", "8"
    ed["Obstacles"]["buildings"] = os.path.join(ROOT, "configs", "buildings.xml")
    if agent is not None:
        ed["Agent"]["xml_path_agent"] = os.path.join(ROOT, "configs", agent)
    ed["Agent"]["Trainer"]["Trainer_path"] = os.path.join(ROOT, "configs", trainer)
    ed.update(kw)
    return ed


class CountTransfers:
    """Counts a learner's get_params / set_params calls: each moves one whole [G][P] vector (one role's, for SAC) between host
    and device."""

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


def make_env(env_golden, env27_golden, n, pool):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=False)
    env.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
    return env


def short_episode_env(env_golden, env27_golden):
    """The golden city and UAV parameters with episodes capped at MAX_STEP steps."""
    city, _, _, _ = city_and_params(env_golden, env27_golden)
    p = env_golden["uav_params"]
    return city, engine.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), MAX_STEP)


# ------------------------------------------------------------------ policy evaluation
def compose(env, n, first, act):
    """uavrl_eval_run / uavrl_sac_eval_run's suite through existing calls: auto-reset with stride N, records on, act on all N rows every iteration."""
    env.set_reset_stride(env.n)
    env.set_records(n)
    env.reset(first)
    obs = env.observe()
    for it in range(100000):
        a, kind = act(obs)
        obs = env.step(a, kind=kind)["obs"]
        if it % 16 == 15 and env.records(clear=False)["slot"].size >= n:
            break
    rec = env.records(clear=False)
    assert list(rec["slot"][:n]) == list(range(n))
    return {k: rec[k][:n] for k in engine.RECORD_FIELDS}


def assert_records_equal(got, want, what):
    for k in engine.RECORD_FIELDS:
        assert_same(got[k], want[k], "%s: %s" % (what, k))


def ring_env(city, params, n, pool, first):
    env = engine.EnvBatch(city, params, n, max_subgoals=64, auto_reset=True)
    env.set_pool(pool["start"], pool["goal"], pool["heading"], pool["sub"], pool["n_sub"])
    env.reset(first)
    return env


# ------------------------------------------------------------------ grouped Q-network trainers
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


def assert_trees_equal(Lg, solo, n_slots):
    leaves, totals, beta = Lg.per_state(n_slots)
    assert leaves.shape == (len(solo), n_slots) and totals.shape == (len(solo),)
    for g, S in enumerate(solo):
        l1, t1, b1 = S.per_state(n_slots)
        assert_same(leaves[g], l1, "leaves of trainer %d" % g)
        assert_same(totals[g:g + 1], np.array([t1]), "total of trainer %d" % g)
        assert beta == b1


# ------------------------------------------------------------------ grouped SAC trainers
def sac(trainers=1, seed=7, **kw):
    kw.setdefault("batch_size", 64)
    return engine.SacLearner(seed=seed, trainers=trainers, **HP, **kw)


def distinct_alphas(S, rng):
    """Every trainer gets its own (log_alpha, exp_avg, exp_avg_sq): a trainer reading another's alpha shows."""
    al = np.stack([[np.log(0.01) + 0.3 * g, 1e-3 * (g + 1), 1e-6 * (g + 2)] for g in range(S.G)]).astype(np.float32)
    al += rng.normal(0, 1e-4, al.shape).astype(np.float32) * np.array([1, 0, 0], np.float32)
    S.set_alpha(al)
    return al


def sac_standalone_like(grouped, g, seed=7, **kw):
    """Trainer g of `grouped` as a stand-alone learner: its parameters, Adam moments, alpha triple and counters, seed + g."""
    s = sac(1, seed + g, **kw)
    for role in range(11):
        s.set_params(role, grouped.get_params(role)[g])
    sc = grouped.scalars()
    s.set_scalars(*grouped.alpha()[g], sc["epoch"], sc["adam_step"])
    return s


def assert_sac_trainers_equal(S, solo, losses=None, solo_losses=None):
    for role in range(SAC_ROLES):
        allp = S.get_params(role).reshape(S.G, -1)
        for g, X in enumerate(solo):
            assert_same(allp[g], X.get_params(role), "role %d of trainer %d" % (role, g))
    al = S.alpha()
    for g, X in enumerate(solo):
        assert_same(al[g], X.alpha()[0], "alpha triple of trainer %d" % g)
        sg, sx = S.scalars(), X.scalars()
        assert (sg["epoch"], sg["adam_step"]) == (sx["epoch"], sx["adam_step"])
    if losses is not None:
        for g in range(len(solo)):
            assert_same(losses[4 * g:4 * g + 4], solo_losses[g], "losses of trainer %d" % g)
