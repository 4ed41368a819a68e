"""CPU-side logic test: csrc/env_core.cuh (the source the CUDA kernel instantiates per env),
compiled for the host by tests/host_shim, against the golden vectors of the Python reference.

Catches step-logic mistakes without a GPU.  The product library is not involved."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
from conftest import episode, ROOT
from env_core_shim import shim, shim_step  # noqa: F401  (module fixture)

@pytest.mark.parametrize("which", ["continuous", "discrete27"])
def test_env_core_matches_reference_goldens(shim, env_golden, env27_golden, which):
    g = env_golden if which == "continuous" else env27_golden
    d = env_golden["dims"]
    city = O.OracleCity(d[0], d[1], d[2], env_golden["buildings"])
    p = env_golden["uav_params"]
    params = O.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    mode = 0 if which == "continuous" else 1
    steps = 0
    for i in range(int(g["epn_episodes"])):
        ep = episode(g, i)
        b = O.OracleBatch(city, params, 1, ep["sub"].shape[0])
        b.reset(ep["start"][None], ep["goal"][None], [ep["heading"]], ep["sub"][None], [ep["n_sub"]], [ep["alias0"]])
        _, _, _, _, obs = shim_step(shim, city, params, b, None, mode)
        np.testing.assert_array_equal(obs[0], ep["obs0"].astype(np.float32))
        for t in range(len(ep["action"])):
            rew, done, info, coll, obs = shim_step(shim, city, params, b, [ep["action"][t]], mode)
            assert abs(rew[0] - ep["reward"][t]) <= 1e-12 * max(1.0, abs(ep["reward"][t])), (i, t)
            assert (done[0], info[0], coll[0]) == (ep["done_ret"][t], ep["info"][t], ep["collision"][t]), (i, t)
            for k in ("px", "py", "pz", "vx", "vy", "V"):
                assert abs(getattr(b, k)[0] - ep[k][t]) <= 1e-12 * max(1.0, abs(ep[k][t])), (i, t, k)
            assert b.step[0] == ep["step"][t] and b.cursor[0] == ep["cursor"][t] and b.done[0] == ep["done"][t]
            np.testing.assert_allclose(obs[0], ep["obs"][t].astype(np.float32), rtol=0, atol=1e-6)
            assert np.array_equal(obs[0, 11:86], ep["obs"][t][11:86]) and np.array_equal(obs[0, 90:95], ep["obs"][t][90:95])
            steps += 1
    assert steps > 1000


@pytest.mark.parametrize("prefix,mode", [("c_", 0), ("d_", 1)])
def test_env_core_single_steps_next_to_every_decision_boundary(shim, env_golden, env27_golden, prefix, mode):
    """The kernel's per-env source (host compile) on the constructed-state single steps of step_golden.npz."""
    from conftest import check_step_outputs, step_batch
    g = np.load(os.path.join(ROOT, "tests", "golden", "step_golden.npz"))
    d = env_golden["dims"]
    city = O.OracleCity(d[0], d[1], d[2], env_golden["buildings"])
    p = env_golden["uav_params"]
    params = O.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    b, n = step_batch(g, prefix, city, params)
    rew, done, info, coll, obs = shim_step(shim, city, params, b, g[prefix + "action"].astype(np.float64), mode)
    check_step_outputs(g, prefix, b, rew, done, info, coll, obs32=obs, exact=False)


def test_env_core_apf_matches_reference_goldens(shim):
    """The kernel's APF source (step_core_apf + apf_force + the queue shift of env_block.cuh's phase 1b, host compile) on the 1 750
    steps of the unmodified reference UAV with APF_Enabled = 1 over obstacles that carry a velocity (tests/golden/apf_golden.npz):
    masks, counters and the whole shifted sub-goal queue exact, fp64 state / reward to 1e-12 (sincos / atan2 of the host libm),
    occupancy bits exact."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "apf_golden.npz"))
    d = g["dims"]
    city = O.OracleCity(d[0], d[1], d[2], g["buildings"])
    p = g["uav_params"]
    params = O.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    ov = np.ascontiguousarray(g["obstacle_v"], np.float64)
    total = 0
    for i in range(int(g["epn_episodes"])):
        ep = episode(g, i)
        b = O.OracleBatch(city, params, 1, ep["sub"].shape[0])
        b.reset(ep["start"][None], ep["goal"][None], [ep["heading"]], ep["sub"][None], [ep["n_sub"]], [ep["alias0"]])
        for t in range(len(ep["action"])):
            rew = np.zeros(1); done = np.zeros(1, np.uint8); info = np.zeros(1, np.uint8); coll = np.zeros(1, np.uint8)
            obs = np.zeros((1, 100), np.float32)
            st = b._struct()
            acts = np.ascontiguousarray([ep["action"][t]], np.float64)
            shim.shim_step_apf(C.c_double(city.c.width), C.c_double(city.c.h), C.c_int(city.buildings.shape[0]),
                               O._p(city.buildings, C.c_double), O._p(ov, C.c_double), C.c_double(params.max_v), C.c_double(params.min_v),
                               C.c_double(params.steering), C.c_double(params.climb_rate), C.c_int(params.max_step), C.c_int(0),
                               C.byref(st), O._p(acts, C.c_double), O._p(rew, C.c_double), O._p(done, C.c_uint8), O._p(info, C.c_uint8),
                               O._p(coll, C.c_uint8), O._p(obs, C.c_float))
            assert abs(rew[0] - ep["reward"][t]) <= 1e-12 * max(1.0, abs(ep["reward"][t])), (i, t, rew[0], ep["reward"][t])
            assert (done[0], info[0], coll[0]) == (ep["done_ret"][t], ep["info"][t], ep["collision"][t]), (i, t)
            for k in ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len"):
                assert abs(getattr(b, k)[0] - ep[k][t]) <= 1e-12 * max(1.0, abs(ep[k][t])), (i, t, k)
            assert b.step[0] == ep["step"][t] and b.cursor[0] == ep["cursor"][t] and b.done[0] == ep["done"][t]
            nleft = int(b.n_sub[0] - b.cursor[0])
            np.testing.assert_allclose(b.sub[0, b.cursor[0]:b.n_sub[0]], ep["subq"][t][:nleft], rtol=0, atol=1e-11, err_msg=str((i, t)))
            np.testing.assert_allclose(obs[0], ep["obs"][t].astype(np.float32), rtol=0, atol=1e-6)
            assert np.array_equal(obs[0, 11:86], ep["obs"][t][11:86]) and np.array_equal(obs[0, 90:95], ep["obs"][t][90:95])
            total += 1
    assert total == 1750


def test_env_core_fly_power_kat(shim):
    """The kernel's fly_power (host compile) vs Agents/UAV.py:241-245 evaluated with Python float arithmetic as written there
    (`**` = libm pow; the kernel forms V**2, V**3, V**4 by repeated multiplication -- within an ulp of pow each, which the cancellation in
    sqrt(1 + V^4 / 4 v0^4) - V^2 / 2 v0^2 amplifies at high speed: 1e-14 relative is asserted, the oracle's libm version is exact),
    constants of config/UAV.xml <Fly_power>."""
    import math
    shim.shim_fly_power.restype = C.c_double
    shim.shim_fly_power.argtypes = [C.c_double] * 10
    P_i, v_0, d_0, rho, s, A, P_b, F_b = 89.0, 4.05, 0.6, 1.225, 0.05, 0.5, 79.0, 120.0
    for j in (0, 1, 3):
        xi, Aj = 0.8 + 0.02 * j, A + 0.03 * j
        for V in (0.0, 0.6, 0.8, 1.0, 2.5, 7.0, 15.0, 30.0):
            induced = P_i * math.sqrt(math.sqrt(1 + (V ** 4) / (4 * (v_0 ** 4))) - (V ** 2) / (2 * (v_0 ** 2)))
            parasite = 0.5 * d_0 * rho * s * Aj * (V ** 3)
            blade = xi * P_b * (1 + 3 * (V ** 2) / (F_b ** 2))
            want = induced + parasite + blade
            got = shim.shim_fly_power(V, P_i, v_0, d_0, rho, s, Aj, P_b, F_b, xi)
            assert abs(got - want) <= 1e-14 * abs(want), (j, V, got, want)
