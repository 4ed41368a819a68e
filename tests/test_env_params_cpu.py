"""The step off the shipped UAV parameters, without a GPU: the CPU oracle and the kernel's per-env source (csrc/env_core.cuh,
host compile) against tests/golden/env_params_golden.npz -- the unmodified reference UAV on a generated 360 x 420 x 60 city
with Steering_angle pi and continuous actions in [-3, 3] (headings far outside one 2 pi wrap), and with Min_V 0 under
discrete-27 actions (zero V_vector with signed zeros).  Every integer output exact, fp64 state and reward to 1e-12, real
observation entries to 1e-6, occupancy bits exact."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
from conftest import GOLDEN, episode
from env_core_shim import shim, shim_step  # noqa: F401  (module fixture: the host compile of env_core.cuh)

F64 = ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLDEN, "env_params_golden.npz"))


def city_params(g, pset):
    d = g["dims"]
    p = g["params"][pset]
    return O.OracleCity(d[0], d[1], d[2], g["buildings"]), O.UavParams(p[0], p[1], p[2], p[4], int(p[3]))


def replay(g, stepper, pset=None):
    """Step every golden episode (of parameter set pset) with stepper(city, params, batch, action, mode) -> (rew, done, info,
    coll, obs32) and compare."""
    n_steps = n_turns = n_still = 0
    for i in range(int(g["epn_episodes"])):
        ep = episode(g, i)
        if pset is not None and int(ep["pset"]) != pset:
            continue
        city, params = city_params(g, int(ep["pset"]))
        mode = int(ep["mode"])
        b = O.OracleBatch(city, params, 1, ep["sub"].shape[0])
        b.reset(ep["start"][None], ep["goal"][None], [ep["heading"]], ep["sub"][None], [ep["n_sub"]], [ep["alias0"]])
        assert (b.vx[0], b.vy[0], b.V[0]) == (ep["vx0"], ep["vy0"], ep["V0"])
        for t in range(len(ep["action"])):
            w = "ep%d t%d" % (i, t)
            rew, done, info, coll, obs = stepper(city, params, b, ep["action"][t], mode)
            assert (done[0], info[0], coll[0]) == (ep["done_ret"][t], ep["info"][t], ep["collision"][t]), w
            assert (b.step[0], b.cursor[0], b.done[0]) == (ep["step"][t], ep["cursor"][t], ep["done"][t]), w
            assert abs(rew[0] - ep["reward"][t]) <= 1e-12 * max(1.0, abs(ep["reward"][t])), (w, rew[0], ep["reward"][t])
            for k in F64:
                assert abs(getattr(b, k)[0] - ep[k][t]) <= 1e-12 * max(1.0, abs(ep[k][t])), (w, k)
            want = ep["obs"][t]
            np.testing.assert_allclose(obs[0], want.astype(np.float32), rtol=0, atol=1e-6, err_msg=w)
            assert np.array_equal(obs[0, 11:86], want[11:86]) and np.array_equal(obs[0, 90:95], want[90:95]), w
            n_steps += 1
            n_turns += int(mode == 0 and abs(ep["action"][t] * params.steering) >= np.pi)
            n_still += int(ep["V"][t] == 0.0)
    return n_steps, n_turns, n_still


def test_golden_covers_what_it_is_for(g):
    """The fixture reaches the branches it exists for: turns of pi or more, zero speed with vx = -0, pops, collisions, lose."""
    vx_neg0 = n_pop = n_coll = n_lose = 0
    for i in range(int(g["epn_episodes"])):
        ep = episode(g, i)
        vx_neg0 += int(((ep["V"] == 0) & np.signbit(ep["vx"])).sum())
        n_pop += int((np.diff(np.r_[0, ep["cursor"]]) > 0).sum())
        n_coll += int(ep["collision"].sum()); n_lose += int((ep["info"] == 2).sum())
    assert vx_neg0 >= 10 and n_pop >= 10 and n_coll >= 5 and n_lose >= 10
    assert g["buildings"][:, 2].min() > 0 and g["dims"][0] != g["dims"][1]


def test_oracle_matches_reference_off_the_shipped_parameters(g):
    def step(city, params, b, a, mode):
        return b.step_(np.array([a]), mode)
    n, turns, still = replay(g, step)
    assert n > 350 and turns > 30 and still > 30


@pytest.mark.parametrize("pset", [0, 1], ids=["steering_pi", "min_v_0"])
def test_env_core_matches_reference_off_the_shipped_parameters(g, shim, pset):  # noqa: F811
    """The kernel's step source.  steering_pi: obs[7] (the cached heading) after turns of up to 3 pi.  min_v_0: the
    0.2 cos|tri_goal - tri_V| term with a zero V_vector (direction (-1, 0) when vx is -0)."""
    def step(city, params, b, a, mode):
        return shim_step(shim, city, params, b, [a], mode)
    n, turns, still = replay(g, step, pset)
    assert n > 150 and (turns > 30 if pset == 0 else still > 30)


def test_negative_min_v_is_refused():
    """A negative Min_V makes the discrete-27 speed negative, which turns V_vector against the heading the step carries:
    uavrl_env_create refuses it (before it looks for a device), like Max_V >= 7."""
    from uavrl_b200 import _lib
    L = _lib.lib()
    b = np.zeros((1, 5))

    def create(max_v, min_v):
        cfg = _lib.EnvConfig()
        cfg.n_envs, cfg.max_subgoals, cfg.max_step = 4, 8, 10
        cfg.len, cfg.width, cfg.h = 500.0, 500.0, 100.0
        cfg.max_v, cfg.min_v, cfg.steering_angle, cfg.climb_rate = max_v, min_v, 0.5, 1.0
        cfg.n_buildings, cfg.buildings_host = 1, b.ctypes.data_as(C.POINTER(C.c_double))
        h = C.c_void_p()
        rc = L.uavrl_env_create(C.byref(cfg), C.byref(h))
        if rc == 0:
            L.uavrl_env_destroy(h)
        return rc, L.uavrl_last_error()
    for min_v in (-0.5, -1e-300, float("nan")):
        rc, msg = create(1.0, min_v)
        assert rc == -1 and b"min_v must be >= 0" in msg, (min_v, rc, msg)
    rc, msg = create(7.0, 0.6)
    assert rc == -1 and b"max_v must be < 7" in msg
    rc, msg = create(1.0, 0.0)                   # Min_V 0 is valid: it reaches the device check (or succeeds on a GPU)
    assert rc == 0 or (rc == -2 and b"no CUDA device" in msg), (rc, msg)
