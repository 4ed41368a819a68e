"""The SAC lockstep loop's refusals, and the kernels one loop iteration launches for each learner.

uavrl_sac_train_run refuses what uavrl_train_run refuses, before it enqueues anything and leaving env, ring and counters as
they were: a learner whose ring rows are not the 100-float observation the env step writes (obs_dim != 100), a learner
without a ring or with lockstep_envs != env.n_envs, an env that was never reset, and an env and learner on different devices.
The launch counts pin which kernels an iteration launches: get_action and the env step, then one update's kernels."""
import pytest
import torch

from gpu_util import city_and_params, sac
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
N, B = 64, 64


@pytest.fixture(scope="module")
def world(env_golden, env27_golden):
    return city_and_params(env_golden, env27_golden)[:2]


def make_env(world, reset=True):
    city, params = world
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=True)
    sc = env.make_scenarios(256, seed=8)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    if reset:
        env.reset(0)
    return env


def assert_refused(call, code, match, S):
    """call() raises UavrlError with `code` and a message matching `match`, launches no kernel, and S keeps its ring and epoch."""
    torch.cuda.synchronize()
    before = (_lib.launch_count(), S.replay_size(), S.scalars()["epoch"])
    with pytest.raises(engine.UavrlError, match=r"uavrl error %d: .*%s" % (code, match)):
        call()
    assert (_lib.launch_count(), S.replay_size(), S.scalars()["epoch"]) == before


REFUSALS = {                    # case: (SacLearner arguments, error code, message)
    "obs64": (dict(obs_dim=64, lockstep_envs=N), ERR_INVALID, "must be 100"),
    "obs96": (dict(obs_dim=96, lockstep_envs=N), ERR_INVALID, "must be 100"),
    "obs124": (dict(obs_dim=124, lockstep_envs=N), ERR_INVALID, "must be 100"),
    "lockstep-mismatch": (dict(lockstep_envs=N // 2), ERR_INVALID, "lockstep_envs must equal env.n_envs"),
    "no-ring": (dict(lockstep_envs=0), ERR_INVALID, "lockstep_envs must equal env.n_envs"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_sac_loop_refusals(world, case):
    """A ring whose rows are not the observation (the env step would write N x 100 floats into frames of N x obs_dim), or a
    ring that is missing or sized for another env count: refused with and without updates, nothing launched or counted."""
    kw, code, match = REFUSALS[case]
    env = make_env(world)
    S = sac(replay_capacity=N * 8, **kw)
    S.init_params(0)
    for do_update in (False, True):
        assert_refused(lambda: engine.sac_train_run(env, S, 3, do_update=do_update), code, match, S)
    env.close(); S.close()


def test_sac_loop_refuses_env_before_reset(world):
    env = make_env(world, reset=False)
    S = sac(replay_capacity=N * 8, lockstep_envs=N)
    S.init_params(0)
    assert_refused(lambda: engine.sac_train_run(env, S, 3), ERR_STATE, "uavrl_sac_train_run before uavrl_env_reset", S)
    env.close(); S.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sac_loop_refuses_device_mismatch(world):
    """An env on device 0 and a SAC learner on device 1: refused with uavrl_train_run's message, nothing launched."""
    env = make_env(world)
    S = sac(replay_capacity=N * 8, lockstep_envs=N, device=1)
    assert_refused(lambda: engine.sac_train_run(env, S, 3), ERR_INVALID, "env and learner live on different devices", S)
    env.close(); S.close()


# ------------------------------------------------------------------ launches per iteration
def launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0, out


def test_sac_iteration_launches(world):
    """Collection only: get_action and the env step.  With an update: also the target, critic, two critic Adam steps, actor,
    actor Adam step and finish kernels."""
    env = make_env(world)
    S = sac(replay_capacity=N * 8, lockstep_envs=N)
    S.init_params(0)
    engine.sac_train_run(env, S, 1, do_update=False)           # observes frame 0; the ring holds N = B transitions
    n, st = launches(lambda: engine.sac_train_run(env, S, 1, do_update=False))
    assert (n, st.updates) == (2, 0)
    n, st = launches(lambda: engine.sac_train_run(env, S, 1))
    assert (n, st.updates) == (9, 1)
    env.close(); S.close()


QNET_ROUTES = {                 # route: (network, launches of an iteration with an update)
    "tc": ((100, [64, 64], 27, False), 5),                     # act, env step, training kernel with the TD pass, dW, Adam
    "fp32": ((100, [128, 64, 64], 27, True), 4),               # act, env step, update kernel, Adam
}


@pytest.mark.parametrize("route", list(QNET_ROUTES))
def test_qnet_iteration_launches(world, route):
    shape, want = QNET_ROUTES[route]
    env = make_env(world)
    L = engine.Learner(*shape, engine.ALGO_DDQN, batch_size=B, replay_capacity=N * 8, lockstep_envs=N, seed=1)
    L.init_params(0)
    r = L.route(B)
    assert (r["tc_train"] is not None and r["td_fused"]) if route == "tc" else (r["tc_fwd"] is None and r["tc_train"] is None)
    engine.train_run(env, L, 1, eps=0.3, do_update=False)
    n, st = launches(lambda: engine.train_run(env, L, 1, eps=0.3, do_update=False))
    assert (n, st.updates) == (2, 0)
    n, st = launches(lambda: engine.train_run(env, L, 1, eps=0.3))
    assert (n, st.updates) == (want, 1)
    env.close(); L.close()
