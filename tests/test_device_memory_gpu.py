"""Device memory ownership: every failing allocation surfaces as "out of memory", frees what the call had taken and leaves the
handle as it was.  uavrl_test_fail_alloc(k) makes the allocation after the next k fail as an exhausted cudaMalloc does, so
each call below is swept over every allocation it makes."""
import gc
import os

import numpy as np
import pytest
import torch

import uavrl_b200  # noqa: F401
from uavrl_b200 import _lib, engine

gpu = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
TOL = 8 << 20                         # bytes of free device memory a balanced call may appear to move
POWER = dict(P_i=89.0, v_0=4.05, d_0=0.6, rho=1.225, s=0.05, A=0.5, P_b=79.0, F_b=120.0, xi=0.8)
N_ENVS, N_SCEN = 64, 16


def fail_alloc(k):
    assert _lib.lib().uavrl_test_fail_alloc(int(k)) == 0


def free_mem():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def city():
    g = np.load(os.path.join(ROOT, "tests", "golden", "env_golden.npz"))
    d, p = g["dims"], g["uav_params"]
    return engine.City(d[0], d[1], d[2], g["buildings"]), engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))


def make_env(extras=False):
    c, p = city()
    env = engine.EnvBatch(c, p, N_ENVS, max_subgoals=64, auto_reset=True)
    try:
        env.set_pool(**env.make_scenarios(N_SCEN, seed=7))
        if extras:
            env.set_extras(power=POWER)
        env.reset(0)
    except Exception:
        env.close()
        raise
    return env


def make_learner(route="tc", trainers=1, lockstep_envs=0, batch_size=32):
    kw = dict(in_dim=99, hidden=[64]) if route == "fp32" else {}
    L = engine.Learner(**kw, batch_size=batch_size, replay_capacity=4096, lockstep_envs=lockstep_envs, trainers=trainers, seed=5)
    L.init_params(3)
    return L


def batch(n, in_dim, seed, sac=False):
    g = torch.Generator().manual_seed(seed)
    s = torch.rand((n, in_dim), generator=g) * 2 - 1
    s2 = torch.rand((n, in_dim), generator=g) * 2 - 1
    a = torch.rand((n, 2), generator=g) * 2 - 1 if sac else torch.randint(0, 27, (n,), generator=g, dtype=torch.int32)
    r = torch.rand(n, generator=g)
    d = (torch.rand(n, generator=g) < 0.1).float()
    return [t.contiguous().cuda() for t in (s, a, r, s2, d)]


def oom_sweep(call, make=None):
    """Sweep call(obj) over its allocations: obj = make() is built with the hook off and kept across k (without make, call
    creates the object and runs once before the sweep, so every kernel it loads is resident).  Every failing k raises "out of
    memory" and leaves no error behind (a probe env steps right after); the first k that succeeds ends the sweep.  Closing
    everything returns free memory to where it was before the sweep: no failing k leaked.  Returns that k."""
    probe = make_env()
    probe_a = torch.zeros(N_ENVS, dtype=torch.int32, device="cuda")
    obj = res = None
    try:
        if make is None:
            call(None).close()
        free_base = free_mem()
        obj = make() if make else None
        k = 0
        while True:
            fail_alloc(k)
            try:
                res = call(obj)
            except engine.UavrlError as e:
                assert "out of memory" in str(e), str(e)
            else:
                break
            finally:
                fail_alloc(-1)
            probe.step(probe_a)
            torch.cuda.synchronize()
            k += 1
            assert k < 200
    finally:
        for o in (res, obj):
            if o is not None and hasattr(o, "close"):
                o.close()
    assert abs(free_mem() - free_base) <= TOL
    probe.close()
    assert k > 0
    return k


# ------------------------------------------------------------------------------------------------- create sweeps
@gpu
def test_env_create_pool_reset_sweep():
    def call(_):
        env = make_env()
        env.observe()
        return env
    oom_sweep(call)


@gpu
@pytest.mark.parametrize("route,trainers", [("tc", 1), ("fp32", 1), ("tc", 4)])
def test_learner_create_sweep(route, trainers):
    def call(_):
        L = make_learner(route, trainers, lockstep_envs=64 if trainers > 1 else 0)
        L.act(torch.zeros((64, L.in_dim), device="cuda"), 0.0)
        return L
    oom_sweep(call)


@gpu
@pytest.mark.parametrize("trainers", [1, 4])
def test_sac_create_sweep(trainers):
    def call(_):
        S = engine.SacLearner(batch_size=32, replay_capacity=4096, lockstep_envs=64, trainers=trainers)
        S.init_params(0)
        S.act(torch.zeros((64, 100), device="cuda"))
        return S
    oom_sweep(call)


@gpu
def test_per_enable_sweep():
    oom_sweep(lambda L: L.per_enable(), make=lambda: make_learner())


@gpu
def test_per_enable_trainers_sweep():
    oom_sweep(lambda L: L.per_enable_trainers(), make=lambda: make_learner(trainers=4, lockstep_envs=64))


@gpu
def test_set_extras_sweep():
    oom_sweep(lambda env: env.set_extras(power=POWER, obstacle_v=np.ones((env.city.buildings.shape[0], 3)), track_envs=8,
                                         track_capacity=256), make=make_env)


@gpu
def test_generate_pool_sweep():
    oom_sweep(lambda env: env.generate_pool(N_SCEN, seed=3), make=make_env)


@gpu
def test_step_host_staging_sweep():
    a = np.zeros(N_ENVS, np.int32)
    obs = np.zeros((N_ENVS, engine.OBS_DIM), np.float32)
    rew, done = np.zeros(N_ENVS, np.float32), np.zeros(N_ENVS, np.uint8)
    oom_sweep(lambda env: env.step_host(a, engine.ACT_DISCRETE27, obs, rew, done), make=make_env)


@gpu
def test_connect_self_sweep():
    oom_sweep(lambda L: L.connect_self(), make=lambda: make_learner())


@gpu
def test_gather_sweep():
    def make():
        L = make_learner()
        s, a, r, s2, d = batch(256, 100, 1)
        L.push(s, a, r, s2, d.to(torch.uint8))
        return L
    oom_sweep(lambda L: L.gather(np.arange(64)), make=make)


@gpu
def test_threaten_rate_sweep():
    pts = np.random.default_rng(0).uniform(0, 100, (500, 3))
    oom_sweep(lambda env: env.threaten_rate(pts), make=make_env)


# ------------------------------------------------------------------------------------------------- state kept
def env_outputs(env, actions):
    out = env.step(actions)
    return [out[k].clone() for k in ("obs", "reward", "done", "info", "collision", "ended")]


@gpu
@pytest.mark.parametrize("what", ["set_pool", "generate_pool", "set_extras"])
def test_failed_state_call_keeps_env(what):
    """After a failed set_pool / generate_pool / set_extras, at every allocation it can fail at, the env steps 50 iterations
    bit-identically to a twin that never made the call: state, reward, observations, sub-goals and energy."""
    env, twin = make_env(extras=True), make_env(extras=True)
    pool = env.make_scenarios(N_SCEN, seed=11)
    nb = env.city.buildings.shape[0]
    calls = {
        "set_pool": lambda: env.set_pool(**pool),
        "generate_pool": lambda: env.generate_pool(N_SCEN, seed=11),
        "set_extras": lambda: env.set_extras(power=POWER, obstacle_v=np.ones((nb, 3)), track_envs=8, track_capacity=256),
    }
    g = torch.Generator().manual_seed(2)
    k = 0
    while True:
        fail_alloc(k)
        try:
            calls[what]()
        except engine.UavrlError as e:
            assert "out of memory" in str(e)
        else:
            break
        finally:
            fail_alloc(-1)
        for _ in range(50):
            a = torch.randint(0, 27, (N_ENVS,), generator=g, dtype=torch.int32).cuda()
            for x, y in zip(env_outputs(env, a), env_outputs(twin, a)):
                assert torch.equal(x, y), k
        s0, s1 = env.get_state(), twin.get_state()
        for key in s0:
            assert np.array_equal(s0[key], s1[key]), (k, key)
        assert np.array_equal(env.get_subgoals(), twin.get_subgoals())
        assert np.array_equal(env.get_energy(), twin.get_energy())
        k += 1
    assert k > 0
    env.close(); twin.close()


# ------------------------------------------------------------------------------------------------- grow failures
def learner_state(L):
    torch.cuda.synchronize()
    return [L.get_params(w) for w in range(5)]


def assert_same(xs, ys, what):
    for i, (x, y) in enumerate(zip(xs, ys)):
        assert np.array_equal(x, y), (what, i)


def grow_sweep(make, fail_call, state, align, check_after):
    """fail_call(obj) grows scratch.  For every k it can fail at: a fresh obj = make() fails with "out of memory" and its state
    (state(obj)) is unchanged; align(obj) resets the counters the failed call advanced, and check_after(obj) (the same call with
    the hook off) must match a twin that never failed."""
    k = 0
    while True:
        obj = make()
        before = state(obj)
        fail_alloc(k)
        try:
            fail_call(obj)
        except engine.UavrlError as e:
            assert "out of memory" in str(e)
        else:
            obj.close()
            break
        finally:
            fail_alloc(-1)
        assert_same(state(obj), before, ("after failure", k))
        align(obj)
        check_after(obj, k)
        obj.close()
        k += 1
    assert k > 0


@gpu
@pytest.mark.parametrize("route", ["tc", "tc-unfused", "fp32"])
def test_learner_grow_failure(route):
    """G = 4, update_batch with 256 rows per trainer against batch_size 32: the partials (and on the tensor-core route the TD and
    row scratch) grow; a failed grow changes no parameter, moment or image, and the next update matches a twin bit for bit."""
    G, Bg = 4, 256
    mk = lambda: make_learner("fp32" if route == "fp32" else "tc", G, lockstep_envs=64)       # noqa: E731
    fuse = route != "tc-unfused"
    _lib.lib().uavrl_set_fuse_td(int(fuse))
    try:
        L0 = mk()
        data = batch(G * Bg, L0.in_dim, 4)
        obs = batch(64, L0.in_dim, 5)[0]
        if route != "fp32":
            assert L0.td_fused(Bg) == fuse
        twin = mk()
        twin.update_batch(*data)
        ref, ref_q = learner_state(twin), twin.act(obs, 0.0, is_train=False, want_q=True)[1].cpu()
        twin.close(); L0.close()

        def state(L):
            return learner_state(L)[:4] + [L.act(obs, 0.0, is_train=False, want_q=True)[1].cpu().numpy()]

        def check_after(L, k):
            L.update_batch(*data)
            assert_same(learner_state(L), ref, ("after the next update", k))
            assert torch.equal(L.act(obs, 0.0, is_train=False, want_q=True)[1].cpu(), ref_q), k

        grow_sweep(mk, lambda L: L.update_batch(*data), state, lambda L: L.set_counters(0, 0), check_after)
    finally:
        _lib.lib().uavrl_set_fuse_td(1)


@gpu
def test_failed_td_grow_keeps_tensor_core_route():
    """A batch too large for the fused TD pass fails at the TD-target (or row) grow; the next update at batch_size, which fuses
    and so grows nothing, still runs the tensor-core training chain and matches a twin that never failed, bit for bit."""
    big = 12000
    large, small = batch(big, 100, 11), batch(32, 100, 12)
    twin = make_learner()
    assert not twin.td_fused(big) and twin.td_fused(32)
    twin.update_batch(*small)
    ref = learner_state(twin)
    twin.close()

    def check_after(L, k):
        r = L.route(32)
        assert r["tc_train"] is not None and r["td_fused"], (k, r)
        L.update_batch(*small)
        assert_same(learner_state(L), ref, ("after the next update", k))

    grow_sweep(make_learner, lambda L: L.update_batch(*large), lambda L: learner_state(L)[:4], lambda L: L.set_counters(0, 0),
               check_after)


@gpu
def test_update_batch_per_grow_failure():
    B = 256
    data = batch(B, 100, 6)
    w = (torch.rand(B, generator=torch.Generator().manual_seed(1)) + 0.5).cuda()
    twin = make_learner()
    err_ref = torch.zeros(B, device="cuda")
    twin.update_batch_per(*data, is_weights=w, abs_err_out=err_ref)
    ref = learner_state(twin)
    twin.close()

    def check_after(L, k):
        err = torch.zeros(B, device="cuda")
        L.update_batch_per(*data, is_weights=w, abs_err_out=err)
        assert_same(learner_state(L), ref, ("after the next update", k))
        assert torch.equal(err, err_ref), k

    grow_sweep(make_learner, lambda L: L.update_batch_per(*data, is_weights=w, abs_err_out=torch.zeros(B, device="cuda")),
               lambda L: learner_state(L)[:4], lambda L: L.set_counters(0, 0), check_after)


@gpu
def test_per_sample_grow_failure():
    def make():
        L = make_learner()
        L.per_enable()
        s, a, r, s2, d = batch(300, 100, 7)
        L.push(s, a, r, s2, d.to(torch.uint8))
        slots = torch.arange(300, dtype=torch.int32, device="cuda")
        L.per_set_errors(slots, torch.rand(300, generator=torch.Generator().manual_seed(3)).cuda())
        return L

    twin = make()
    ref = [t.cpu() for t in twin.per_sample(64)]
    twin.close()

    def state(L):
        leaves, total, beta = L.per_state(L.cfg.replay_capacity)            # every slot of the tree
        return [leaves, np.array([total, beta])]

    def check_after(L, k):
        got = L.per_sample(64)
        assert all(torch.equal(x.cpu(), y) for x, y in zip(got, ref)), k

    grow_sweep(make, lambda L: L.per_sample(64), state, lambda L: None, check_after)


@gpu
def test_sac_grow_failure():
    G, Bg = 4, 256

    def make():
        S = engine.SacLearner(batch_size=32, replay_capacity=4096, trainers=G)
        S.init_params(1)
        return S

    data = batch(G * Bg, 100, 8, sac=True)
    twin = make()
    twin.update_batch(*data)
    torch.cuda.synchronize()
    ref = [twin.get_params(r) for r in range(14)] + [twin.alpha()]
    twin.close()

    def state(S):
        torch.cuda.synchronize()
        return [S.get_params(r) for r in range(11)] + [S.alpha()]

    def align(S):
        sc = S.scalars()
        S.set_scalars(sc["log_alpha"], sc["la_m"], sc["la_v"], 0, 0)

    def check_after(S, k):
        S.update_batch(*data)
        torch.cuda.synchronize()
        assert_same([S.get_params(r) for r in range(14)] + [S.alpha()], ref, ("after the next update", k))

    grow_sweep(make, lambda S: S.update_batch(*data), state, align, check_after)


# ------------------------------------------------------------------------------------------------- real exhaustion, cycles
@gpu
def test_learner_failed_allocation_frees_everything():
    """No hook: the replay ring (4.4e14 bytes) cannot be allocated; the parameters, partials and the scratch sized for a batch
    of 2^24 that were already allocated are freed, and no error is left for the next launch."""
    free0 = free_mem()
    with pytest.raises(engine.UavrlError, match="out of memory"):
        engine.Learner(batch_size=1 << 24, replay_capacity=1 << 40, lockstep_envs=1024)
    assert abs(free_mem() - free0) <= TOL
    L = make_learner()
    L.act(torch.zeros((64, 100), device="cuda"), 0.0)
    torch.cuda.synchronize()
    L.close()


def env_cycle():
    env = make_env()
    env.set_extras(power=POWER, track_envs=8, track_capacity=64)
    env.reset(0)
    env.step_host(np.zeros(N_ENVS, np.int32), engine.ACT_DISCRETE27, np.zeros((N_ENVS, engine.OBS_DIM), np.float32),
                  np.zeros(N_ENVS, np.float32), np.zeros(N_ENVS, np.uint8))
    env.close()


def learner_cycle():
    L = make_learner(trainers=4, lockstep_envs=64)
    L.per_enable_trainers()
    L.update_batch(*batch(4 * 128, 100, 9))
    L.close()


def sac_cycle():
    S = engine.SacLearner(batch_size=32, replay_capacity=4096, lockstep_envs=64, trainers=4)
    S.update_batch(*batch(4 * 128, 100, 10, sac=True))
    S.close()


@gpu
@pytest.mark.parametrize("cycle", [env_cycle, learner_cycle, sac_cycle], ids=["env", "learner", "sac"])
def test_create_destroy_cycles(cycle):
    cycle()
    free0 = free_mem()
    for _ in range(50):
        cycle()
    assert abs(free_mem() - free0) <= TOL
