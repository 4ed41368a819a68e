"""Moving obstacles on the device (uavrl_env_set_motion): the env step against the reference loop (motion_golden.npz) and
against the oracle with the same table rule (motion_oracle.py), the table's read-back, equivalences, the loops and the
refusals."""
import os

import numpy as np
import pytest
import torch

import motion_oracle as MO
import oracle as O
from conftest import ROOT
from gpu_util import assert_close64, assert_obs, city_and_params
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu
K = 64


@pytest.fixture(scope="module")
def mg():
    return np.load(os.path.join(ROOT, "tests", "golden", "motion_golden.npz"))


def velocity(tab, vz):
    v = np.zeros((tab.shape[0], 3))
    v[:, :2] = tab[:, 2:]
    v[:, 2] = vz
    return v


def centres(tab):
    return np.concatenate([tab[:, :2], np.zeros((tab.shape[0], 1))], 1)


def random_city(env_golden, n, seed):
    """n cylinders over the golden city's box (n = 26: the shipped city), and their table with random velocities."""
    rng = np.random.default_rng(seed)
    L, W, H = env_golden["dims"]
    if n == 26:
        b = env_golden["buildings"].copy()
    else:
        b = np.zeros((n, 5))
        b[:, 0] = rng.uniform(0, L, n); b[:, 1] = rng.uniform(0, W, n)
        b[:, 3] = rng.uniform(5, 25, n); b[:, 4] = rng.uniform(10, 60, n)
    tab = np.zeros((n, 4))
    tab[:, :2] = b[:, :2]
    tab[:, 2:] = rng.normal(0, 2.5, (n, 2))
    tab[rng.uniform(size=n) < 0.2, 2:] = 0.0
    return b, tab


def oracle_reset_ended(ob, sc, scen, stride, P, ocity, oparams):
    ended = np.nonzero(ob.done)[0]
    if ended.size:
        scen[ended] = (scen[ended] + stride) % P
        fresh = O.OracleBatch(ocity, oparams, ended.size, K)
        fresh.reset(sc["start"][scen[ended]], sc["goal"][scen[ended]], sc["heading"][scen[ended]], sc["sub"][scen[ended]],
                    sc["n_sub"][scen[ended]])
        for k in ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len", "step", "cursor", "n_sub", "done", "alias0"):
            getattr(ob, k)[ended] = getattr(fresh, k)
        ob.goal[ended] = fresh.goal; ob.sub[ended] = fresh.sub


@pytest.mark.parametrize("c", [0, 1, 2], ids=["continuous", "apf", "discrete27"])
def test_kernel_reproduces_reference_loop(mg, env_golden, env27_golden, c):
    """Every golden episode through the device step with the table set to the reference's after its first run(): masks
    exact, fp64 state to 1e-9, the observation after step k equal to the reference's state_test of iteration k + 1, and the
    table bit for bit."""
    d, p = mg["dims"], mg["uav_params"]
    city = engine.City(d[0], d[1], d[2], mg["buildings"])
    params = engine.UavParams(p[0], p[1], p[2], float(mg["climb_rate"]), int(p[3]))
    vz = mg["obstacle_v"][:, 2]
    i = 0
    while "cfg%d_ep%d_action" % (c, i) in mg:
        pre = "cfg%d_ep%d_" % (c, i)
        ep = {k[len(pre):]: mg[k] for k in mg.files if k.startswith(pre)}
        env = engine.EnvBatch(city, params, 1, max_subgoals=K)
        env.set_pool(ep["start"][None], ep["goal"][None], [ep["heading"]], ep["sub"][None], [ep["n_sub"]], [ep["alias0"]])
        v = velocity(ep["tab1"], vz)
        if c == 1:
            env.set_extras(obstacle_v=v)
        env.set_motion(v, positions=centres(ep["tab1"]))
        env.reset(0)
        assert_obs(env.observe().cpu().numpy(), ep["state_test"][:1], "obs0")
        kind = engine.ACT_DISCRETE27 if c == 2 else engine.ACT_CONT_F64
        for t in range(len(ep["action"])):
            a = torch.tensor([int(ep["action"][t])], dtype=torch.int32, device="cuda") if c == 2 else \
                torch.tensor([ep["action"][t]], dtype=torch.float64, device="cuda")
            o = {k: x.cpu().numpy() for k, x in env.step(a, kind=kind).items()}
            assert (o["done"][0], o["info"][0], o["collision"][0]) == (ep["done_ret"][t], ep["info"][t], ep["collision"][t]), (c, i, t)
            st = env.get_state()
            assert_close64(st["reward64"], [ep["reward"][t]], 1e-9, "reward")
            for k in ("px", "py", "pz"):
                assert_close64(st[k], [ep[k][t]], 1e-9, k)
            pos, vel, steps = env.obstacles()
            assert steps == t + 1
            if t + 1 < len(ep["action"]):
                tab = np.concatenate([pos[:, :2], vel[:, :2]], 1)
                assert MO.table_digest(tab) == ep["tab_digest"][t + 1].tobytes(), (c, i, t)
                assert_obs(o["obs"], ep["state_test"][t + 1][None], "obs c%d e%d t%d" % (c, i, t))
        env.close()
        i += 1


def run_vs_oracle(env_golden, env27_golden, N, T, nb, apf, mode, seed):
    _, params, _, oparams = city_and_params(env_golden, env27_golden)
    d = env_golden["dims"]
    b, tab = random_city(env_golden, nb, seed)
    vz = np.zeros(nb); vz[::7] = 0.25
    city = engine.City(d[0], d[1], d[2], b)
    env = engine.EnvBatch(city, params, N, max_subgoals=K, auto_reset=True)
    P = max(2 * N, 64)
    sc = env.make_scenarios(P, seed=seed)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    v = velocity(tab, vz)
    if apf:
        env.set_extras(obstacle_v=v)
    env.set_motion(v, positions=centres(tab))
    env.reset(0)
    mc = MO.MovingCity(d[0], d[1], d[2], b, tab, vz, apf=apf)
    try:
        ob = O.OracleBatch(mc.city, oparams, N, K)
        scen = np.arange(N) % P
        ob.reset(sc["start"][scen], sc["goal"][scen], sc["heading"][scen], sc["sub"][scen], sc["n_sub"][scen])
        assert_obs(env.observe().cpu().numpy(), ob.state(want64=True)[1], "obs0")
        rng = np.random.default_rng(seed)
        for t in range(T):
            if mode == "discrete27":
                a = rng.integers(0, 27, N).astype(np.int32)
                out = env.step(torch.tensor(a, device="cuda"))
                rew, done, info, coll, _ = ob.step_(a.astype(np.float64), O.ACT_DISCRETE27, want_obs=False)
            else:
                a = rng.uniform(-1, 1, N)
                out = env.step(torch.tensor(a, device="cuda"), kind=engine.ACT_CONT_F64)
                rew, done, info, coll, _ = ob.step_(a, O.ACT_CONTINUOUS, want_obs=False)
            mc.advance()
            o = {k: x.cpu().numpy() for k, x in out.items()}
            assert np.array_equal(o["done"], done) and np.array_equal(o["info"], info) and np.array_equal(o["collision"], coll), t
            st = env.get_state()
            assert_close64(st["reward64"], rew, 1e-9, "reward t%d" % t)
            oracle_reset_ended(ob, sc, scen, N, P, mc.city, oparams)
            for k in ("px", "py", "pz"):
                assert_close64(st[k], getattr(ob, k), 1e-9, "%s t%d" % (k, t))
            assert_obs(o["obs"], ob.state(want64=True)[1], "obs t%d" % t)
            assert np.array_equal(st["cursor"], ob.cursor) and np.array_equal(st["step"], ob.step), t
            if apf:
                # every queue every step (moving obstacles push sub-goals hard, the aliased entry 0 included); the oracle then
                # continues from the kernel's queues, so a failure points at the step that made it
                subs = env.get_subgoals()
                for e in range(N):
                    c, n = int(ob.cursor[e]), int(ob.n_sub[e])
                    assert_close64(subs[e, c:n], ob.sub[e, c:n], 1e-9, "queue e%d t%d" % (e, t))
                ob.sub[:] = subs
            pos, vel, steps = env.obstacles()
            assert steps == t + 1 and np.array_equal(pos[:, :2], mc.tab[:, :2]) and np.array_equal(vel[:, :2], mc.tab[:, 2:]), t
    finally:
        mc.close()
    return env


@pytest.mark.parametrize("nb,apf,mode", [(26, True, "discrete27"), (26, False, "continuous"), (64, False, "discrete27"),
                                         (64, True, "continuous"), (1, True, "discrete27"), (1, False, "continuous")])
def test_against_oracle_1024_envs_with_auto_reset(env_golden, env27_golden, nb, apf, mode):
    run_vs_oracle(env_golden, env27_golden, 1024, 300, nb, apf, mode, seed=nb + 2 * apf)


@pytest.mark.parametrize("N", [1, 7, 33, "small+1", 20011])
def test_batch_sizes(env_golden, env27_golden, N):
    from uavrl_b200 import _lib as L
    if N == "small+1":
        N = 4 * torch.cuda.get_device_properties(0).multi_processor_count * 8 + 1
    run_vs_oracle(env_golden, env27_golden, N, 40 if N > 1000 else 120, 26, True, "discrete27", seed=5)
    assert L is _lib


def test_observe_and_threaten_rate_read_without_advancing(env_golden, env27_golden):
    env = run_vs_oracle(env_golden, env27_golden, 64, 30, 26, False, "discrete27", seed=9)
    pos, vel, steps = env.obstacles()
    o1 = env.observe().cpu().numpy(); o2 = env.observe().cpu().numpy()
    assert np.array_equal(o1, o2)
    centres = np.stack([pos[:, 0], pos[:, 1], np.full(len(pos), 1.0)], 1)
    assert env.threaten_rate(centres).all()                    # the moved centres are inside their cylinders
    assert env.obstacles()[2] == steps and np.array_equal(env.obstacles()[0], pos)


def test_zero_velocity_equals_motion_off_and_shards(env_golden, env27_golden):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N, W, T = 512, 4, 150
    nb = env_golden["buildings"].shape[0]

    def make(n, motion, first=0):
        env = engine.EnvBatch(city, params, n, max_subgoals=K, auto_reset=True)
        env.generate_pool(2048, seed=3)
        if motion is not None:
            env.set_motion(motion)
        env.set_reset_stride(N)
        env.reset(first)
        return env
    rng = np.random.default_rng(4)
    acts = [torch.tensor(rng.integers(0, 27, N).astype(np.int32), device="cuda") for _ in range(T)]
    a, b = make(N, None), make(N, np.zeros((nb, 3)))
    for t in range(T):
        oa, ob = a.step(acts[t]), b.step(acts[t])
        for k in oa:
            assert torch.equal(oa[k], ob[k]), (k, t)
    vel = np.random.default_rng(6).normal(0, 2, (nb, 3))
    full = make(N, vel)
    shards = [make(N // W, vel, first=r * N // W) for r in range(W)]
    for t in range(T):
        of = full.step(acts[t])
        os_ = [s.step(acts[t][r * N // W:(r + 1) * N // W]) for r, s in enumerate(shards)]
        for k in of:
            assert torch.equal(of[k], torch.cat([o[k] for o in os_])), (k, t)
    for s in shards:
        assert all(np.array_equal(x, y) for x, y in zip(s.obstacles(), full.obstacles()))


@pytest.mark.parametrize("sac", [False, True])
def test_training_loops_advance_once_per_iteration(env_golden, env27_golden, sac):
    """train_run / sac_train_run with motion: one table run per iteration, the same launch count per iteration as without
    motion, identical results with dependent launches on and off, and ring frame t + 1 = the observation on O_{t+1}."""
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    N, T = 256, 12
    nb = env_golden["buildings"].shape[0]
    vel = np.random.default_rng(8).normal(0, 2, (nb, 3))

    def run(motion, pdl):
        _lib.lib().uavrl_set_pdl(int(pdl))
        env = engine.EnvBatch(city, params, N, max_subgoals=K, auto_reset=True)
        env.generate_pool(1024, seed=2)
        env.set_records(4096)                                  # the extras step both with and without motion
        if motion:
            env.set_motion(vel)
        env.reset(0)
        if sac:
            L = engine.SacLearner(batch_size=64, replay_capacity=16 * N, lockstep_envs=N, seed=1)
            run_fn = lambda n: engine.sac_train_run(env, L, n)  # noqa: E731
        else:
            L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=16 * N, lockstep_envs=N)
            L.init_params(0)
            run_fn = lambda n: engine.train_run(env, L, n, eps=0.2)  # noqa: E731
        run_fn(2)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        run_fn(T)
        torch.cuda.synchronize()
        return env, (_lib.launch_count() - c0) / T, env.get_state(), env.observe().cpu().numpy()
    try:
        env_on, per_on, st_on, obs_on = run(True, True)
        _, per_off, _, _ = run(False, True)
        _, per_on2, st_on2, obs_on2 = run(True, False)
    finally:
        _lib.lib().uavrl_set_pdl(1)
    assert per_on == per_off and env_on.obstacles()[2] == T + 2
    assert np.array_equal(obs_on, obs_on2) and all(np.array_equal(st_on[k], st_on2[k]) for k in st_on)
    tab = np.zeros((nb, 4)); tab[:, :2] = env_golden["buildings"][:, :2]; tab[:, 2:] = vel[:, :2]
    for _ in range(T + 2):
        MO.obstacle_run(tab, env_golden["dims"][0], env_golden["dims"][1])
    pos, v, _ = env_on.obstacles()
    assert np.array_equal(pos[:, :2], tab[:, :2]) and np.array_equal(v[:, :2], tab[:, 2:])


def test_refusals_and_failed_allocations_change_nothing(env_golden, env27_golden):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    L, Wd = env_golden["dims"][0], env_golden["dims"][1]
    nb = env_golden["buildings"].shape[0]
    env = engine.EnvBatch(city, params, 64, max_subgoals=K, auto_reset=True)
    env.generate_pool(256, seed=1)
    vel = np.random.default_rng(1).normal(0, 2, (nb, 3))
    env.set_extras(obstacle_v=vel)
    env.set_motion(vel)
    env.reset(0)
    for _ in range(5):
        env.step(torch.zeros(64, dtype=torch.int32, device="cuda"))
    before = env.obstacles(), env.get_state(), env.get_subgoals()
    bad_pos = env_golden["buildings"][:, :3].copy()
    bad = [dict(velocity=np.where(np.arange(nb * 3).reshape(nb, 3) == 4, np.nan, vel)),
           dict(velocity=vel, positions=np.where(np.arange(nb * 3).reshape(nb, 3) == 0, -1.0, bad_pos)),
           dict(velocity=vel, positions=np.where(np.arange(nb * 3).reshape(nb, 3) == 1, Wd + 1.0, bad_pos)),
           dict(velocity=np.where(np.arange(nb * 3).reshape(nb, 3) == 0, L + 1.0, vel)),
           dict(velocity=vel * 0.5)]                            # differs from the APF model's obstacle_v
    for kw in bad:
        with pytest.raises(engine.UavrlError):
            env.set_motion(**kw)
    with pytest.raises(engine.UavrlError):
        env.set_extras(obstacle_v=vel * 2)                      # differs from the motion table
    for k in range(3):
        _lib.lib().uavrl_test_fail_alloc(k)
        try:
            with pytest.raises(engine.UavrlError):
                env.set_motion(vel)
        finally:
            _lib.lib().uavrl_test_fail_alloc(-1)
    after = env.obstacles(), env.get_state(), env.get_subgoals()
    assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0]))
    assert all(np.array_equal(before[1][k], after[1][k]) for k in before[1]) and np.array_equal(before[2], after[2])
    env.step(torch.zeros(64, dtype=torch.int32, device="cuda"))
    assert env.obstacles()[2] == before[0][2] + 1
    env.set_motion(None)
    assert env.obstacles()[2] == 0 and not env.obstacles()[1].any()


def test_eval_run_repeats_from_a_restored_table(env_golden, env27_golden):
    city, params, _, _ = city_and_params(env_golden, env27_golden)
    nb = env_golden["buildings"].shape[0]
    vel = np.random.default_rng(3).normal(0, 2, (nb, 3))
    env = engine.EnvBatch(city, params, 128, max_subgoals=K, auto_reset=True)
    env.generate_pool(512, seed=4)
    env.reset(0)
    L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=1024, lockstep_envs=128)
    L.init_params(0)
    recs = []
    for _ in range(2):
        env.set_motion(vel, positions=env_golden["buildings"][:, :3])
        r = engine.eval_run(env, L, 256, first_scenario=0)
        recs.append(r)
        assert env.obstacles()[2] > 0
    a, b = recs
    assert a["n_records"] == b["n_records"] > 0
    for k in a["records"]:
        assert np.array_equal(np.asarray(a["records"][k]), np.asarray(b["records"][k])), k
