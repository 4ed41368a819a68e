"""Env sweep: the CUDA step / observation kernel against the CPU oracle across cities, UAV parameters, sub-goal capacities,
batch sizes, action kinds and the optional models -- the inputs uavrl_env_create accepts beyond the shipped configuration
that test_env_gpu.py runs.  Each row runs engine.EnvBatch and oracle.OracleBatch side by side for a few dozen steps with the
tolerances of test_env_gpu.py: every integer output exact (done, info, collision, ended, step, cursor, scenario, occupancy
bits), fp64 state and reward 1e-9 relative, real observation entries 1e-5.  Cities are generated from a seed.  Each row
asserts the branches it exists for with counters (collisions, sub-goal pops, lose, success, in-kernel restarts).

The oracle is pinned to the reference off the shipped parameters by tests/golden/env_params_golden.npz
(test_env_params_cpu.py); the last test here runs the kernel on that golden too."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

import oracle as O
from conftest import GOLDEN, episode
from env_sweep import (CITIES, F64, KIND, POWER, assert_obs_heading_on_circle, cities, fly_power, hand_pool, make_city,
                       oracle_auto_reset, params_of, seek, small_batch_envs)
from gpu_util import assert_close64, assert_obs

pytestmark = pytest.mark.gpu

def run_row(city_kind, N, K, params_kw, kind="d27", bound=1.0, T=30, auto_reset=True, P=None, pool_kw=None, age=(None, None),
            extras=None, seed=0, obs_every=1):
    """Step the CUDA env and the oracle side by side; returns counters of the branches taken."""
    from uavrl_b200 import _lib, engine
    city, ocity = cities(city_kind)
    params, oparams = engine.UavParams(**params_kw), O.UavParams(**params_kw)
    rng = np.random.default_rng(seed)
    P = P or max(2 * N, 16)
    sc = hand_pool(ocity, P, K, rng, **(pool_kw or {}))
    env = engine.EnvBatch(city, params, N, max_subgoals=K, auto_reset=auto_reset)
    apf_v = None
    try:
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
        if extras:
            env.set_extras(**extras)
            apf_v = extras.get("obstacle_v")
        env.reset(0)
        scen = np.arange(N) % P
        ob = O.OracleBatch(ocity, oparams, N, K)
        ob.reset(sc["start"][scen], sc["goal"][scen], sc["heading"][scen], sc["sub"][scen], sc["n_sub"][scen], sc["alias0"][scen])
        O.set_apf(apf_v)
        assert_obs(env.observe().cpu().numpy(), ob.state(want64=True)[1], "obs0")
        cnt = dict(coll=0, pop=0, lose=0, success=0, restart=0, steps=0)
        kname, tdt = KIND[kind]
        energy = np.zeros(N)
        for t in range(T):
            a = seek(ob, oparams, rng, kind, bound)
            if kind == "f32x2":
                a2 = np.stack([a.astype(np.float32), rng.uniform(-9, 9, N).astype(np.float32)], 1)    # only [.., 0] steers
                act, a64 = torch.tensor(a2, device="cuda"), a2[:, 0].astype(np.float64)
            elif kind == "f32":
                act, a64 = torch.tensor(a.astype(np.float32), device="cuda"), a.astype(np.float32).astype(np.float64)
            else:
                act, a64 = torch.tensor(a, dtype=tdt, device="cuda"), a.astype(np.float64)
            cur_before = ob.cursor.copy()
            out = env.step(act, kind=getattr(_lib, kname))
            rew, done, info, coll, _ = ob.step_(a64, O.ACT_DISCRETE27 if kind == "d27" else O.ACT_CONTINUOUS, want_obs=False)
            o = {k: v.cpu().numpy() for k, v in out.items()}
            w = "t%d" % t
            assert np.array_equal(o["done"], done) and np.array_equal(o["info"], info), w
            assert np.array_equal(o["collision"], coll) and np.array_equal(o["ended"], ob.done), w
            np.testing.assert_allclose(o["reward"], rew, rtol=1e-5, atol=1e-5)
            st = env.get_state()
            assert_close64(st["reward64"], rew, 1e-9, "reward " + w)
            if extras and "power" in extras:
                # + Calc_Fly_Power(V) of this step (the oracle has not restarted yet); an ended env restarts with 0
                energy = np.where(ob.done.astype(bool), 0.0, energy + np.array([fly_power(v) for v in ob.V]))
                ended_last = ob.done.astype(bool).copy()
            cnt["pop"] += int(((ob.cursor > cur_before) & (info == 1)).sum())
            if auto_reset:
                cnt["restart"] += oracle_auto_reset(ob, sc, scen, N, P, ocity, oparams, K)
                assert np.array_equal(st["scenario"], scen), w
            assert np.array_equal(st["step"], ob.step) and np.array_equal(st["cursor"], ob.cursor), w
            assert np.array_equal(st["done"], ob.done), w
            for k in F64:
                assert_close64(st[k], getattr(ob, k), 1e-9, k + " " + w)
            if t % obs_every == 0 or t == T - 1:
                assert_obs_heading_on_circle(o["obs"], ob.state(want64=True)[1], "obs " + w)
            if apf_v is not None and t % 5 == 0:
                subs = env.get_subgoals()
                for e in range(0, N, max(1, N // 16)):
                    c, n = int(ob.cursor[e]), int(ob.n_sub[e])
                    assert_close64(subs[e, c:n], ob.sub[e, c:n], 1e-9, "queue e%d %s" % (e, w))
            if extras and "power" in extras:
                np.testing.assert_allclose(env.get_energy(), energy, rtol=1e-12, atol=1e-9)
            cnt["coll"] += int(coll.sum()); cnt["lose"] += int((info == 2).sum()); cnt["success"] += int((info == 1).sum())
            cnt["steps"] += N
            if extras and extras.get("track_envs"):
                for e in range(extras["track_envs"]):       # UAV.path: the position after every step of the episode
                    path = env.get_path(e, 1 if ended_last[e] else 0)
                    assert len(path) and np.array_equal(path[-1], [st["px"][e], st["py"][e], st["pz"][e]]) if not ended_last[e] \
                        else len(path) >= 1, (e, w)
            if t == 0 and age[0] is not None:
                # the first step pops the aliased sub-goal and restarts the segment (Step = 0): age the segments now so
                # that Max_Step ('lose') and the restart happen inside the run
                aged = rng.integers(age[0], age[1], N).astype(np.int32)
                env.set_state(step=aged); ob.step[:] = aged
        return cnt
    finally:
        O.set_apf(None)
        env.close()


# ----------------------------------------------------------------------------------------------------------- the table
# id: (city, N, K, params, kind, bound, T, extra run_row arguments, counters that must be > 0)
ROWS = {
    "city_empty": ("empty", 64, 8, params_of(max_v=3.0, min_v=1.0, max_step=40), "d27", 1, 40, {}, ("pop", "lose")),
    "city_one": ("one", 64, 8, params_of(max_v=2.0, max_step=40), "d27", 1, 40, {}, ("pop", "lose")),
    "city_dense64": ("dense64", 256, 16, params_of(max_v=2.0, max_step=40), "d27", 1, 40, {"pool_kw": {"z": (1.0, 30.0)}},
                     ("coll", "pop", "lose", "restart")),
    "city_box300x800": ("box300x800", 128, 8, params_of(max_v=3.0, min_v=1.0, max_step=40), "f64", 1, 40, {}, ("coll", "pop", "lose")),
    "max_v_6.9": ("dense64", 256, 8, params_of(max_v=6.9, min_v=2.0, max_step=30), "d27", 1, 35, {}, ("coll", "pop", "lose", "restart")),
    "max_v_3_min_v_1": ("box300x800", 96, 8, params_of(max_v=3.0, min_v=1.0, max_step=30), "d27", 1, 35, {}, ("coll", "pop", "lose")),
    # steering 0.5 rad, not pi / 6: a zero V_vector snaps the heading to 0 or pi, and three pi / 6 turns from there end within
    # ulps of pi / 2, where the sign of cos -- and so of the next zero vx -- rests on the last bit of the heading
    "min_v_0": ("dense64", 128, 8, params_of(max_v=2.0, min_v=0.0, steering=0.5, max_step=30), "d27", 1, 35, {},
                ("coll", "pop", "lose")),
    "min_v_above_max_v": ("one", 64, 8, params_of(max_v=1.5, min_v=4.0, max_step=30), "d27", 1, 35, {}, ("coll", "pop", "lose")),
    "climb_0": ("dense64", 96, 8, params_of(climb_rate=0.0, max_step=30), "d27", 1, 35, {}, ("coll", "pop", "lose")),
    "climb_5": ("dense64", 96, 8, params_of(climb_rate=5.0, max_step=30), "d27", 1, 35, {"pool_kw": {"z": (0.5, 12.0)}},
                ("coll", "pop", "lose")),
    "max_step_1": ("one", 64, 8, params_of(max_step=1), "d27", 1, 12, {}, ("lose", "restart")),
    "max_step_2": ("dense64", 64, 8, params_of(max_step=2), "f32", 1, 12, {}, ("lose", "restart")),
    "max_step_5": ("box300x800", 64, 8, params_of(max_v=3.0, max_step=5), "d27", 1, 16, {}, ("lose", "restart", "pop")),
    "K_1_n_sub_1": ("one", 64, 1, params_of(max_v=3.0, max_step=20), "d27", 1, 30, {"pool_kw": {"n_sub": 1}}, ("success", "restart")),
    "K_2_alias": ("empty", 64, 2, params_of(max_v=3.0, max_step=30), "d27", 1, 30, {"pool_kw": {"n_sub": 2, "alias": 1}},
                  ("pop", "success", "restart")),
    "K_2_no_alias": ("dense64", 64, 2, params_of(max_v=3.0, max_step=30), "f64", 1, 30, {"pool_kw": {"n_sub": 2, "alias": 0}},
                     ("pop", "restart")),
    "K_3_alias": ("one", 64, 3, params_of(max_v=3.0, max_step=30), "d27", 1, 30, {"pool_kw": {"n_sub": 3, "alias": 1}},
                  ("pop", "success", "restart")),
    "K_3_no_alias": ("empty", 64, 3, params_of(max_v=3.0, max_step=30), "f32", 1, 30, {"pool_kw": {"n_sub": 3, "alias": 0}},
                     ("pop", "restart")),
    "apf_64_max_v_3": ("apf", 96, 8, params_of(max_v=3.0, max_step=30), "d27", 1, 30, {"apf": True, "pool_kw": {"z": (8.0, 14.0), "near": (250.0, 250.0, 12.0), "alias": 0}},
                       ("coll", "pop", "lose")),
    "energy_tracking": ("dense64", 96, 8, params_of(max_v=4.0, min_v=0.5, max_step=20), "d27", 1, 30,
                        {"extras": {"power": POWER, "track_envs": 8, "track_capacity": 64}}, ("coll", "pop", "lose", "restart")),
}
for _kind in ("f64", "f32", "f32x2"):
    for _name, _st in (("pi_2", np.pi / 2), ("pi", np.pi)):
        ROWS["steering_%s_%s" % (_name, _kind)] = ("dense64", 128, 8, params_of(max_v=2.0, steering=_st, max_step=30), _kind, 3, 35, {},
                                                   ("coll", "pop", "lose"))


@pytest.mark.parametrize("row", sorted(ROWS))
def test_row_against_oracle(row):
    """One configuration row.  The min_v_0 and steering_pi_* rows failed before the heading and zero-velocity fixes
    (obs[7] outside [0, 2 pi]; the 0.2 cos|tri_goal - tri_V| term of a zero V_vector with the wrong sign).  The APF row's
    pools do not alias sub_goals[0] to the position: a force of 7 m or more keeps that entry from being popped on the first
    step, and the kernel does not store the moved entry back into the queue (the deviation env.cu documents for Max_V >= 7)."""
    city, N, K, params, kind, bound, T, kw, need = ROWS[row]
    kw = dict(kw)
    if kw.pop("apf", False):
        rng = np.random.default_rng(5)
        nb = make_city(city)[3].shape[0]
        vel = np.zeros((nb, 3)); vel[:, :2] = rng.normal(0, 1.5, (nb, 2)); vel[::7] = 0.0          # some static: skipped
        kw["extras"] = {"obstacle_v": vel}
    age = (max(0, params["max_step"] - 12), params["max_step"]) if params["max_step"] > 12 else (None, None)
    cnt = run_row(city, N, K, params, kind=kind, bound=bound, T=T, age=age, seed=zlib.crc32(row.encode()) % 1000, **kw)
    for k in need:
        assert cnt[k] > 0, (row, cnt)


def test_apf_early_return_is_reached():
    """The apf city's disc stack: at a UAV height of 10 m over the centre more than 50 obstacles have the point inside their
    3-D radius, each adding at least 2 to UAV.cal_force's running magnitude -- the documented `cum > 100` return is taken
    (the oracle returns there too, and test_row_against_oracle[apf_64_max_v_3] flies over it)."""
    b = make_city("apf")[3]
    d = np.sqrt((b[:, 0] - 250) ** 2 + (b[:, 1] - 250) ** 2 + (10 - b[:, 2]) ** 2) - b[:, 3]
    assert (d < 0).sum() > 50


@pytest.mark.parametrize("N", ["1", "7", "8", "9", "31", "33", "small-1", "small", "small+1", "20011"])
def test_batch_sizes_and_cta_shapes(N):
    """Ragged last CTAs of both kernel shapes.  N <= small_batch_envs() (4 * SMs * 8, 4 224 on 132 SMs) runs
    env_kernel<true, 8>, N above it env_kernel<true, 32>: small-1 and small run the 8-env CTAs, small+1 and 20 011 (above
    16 384, not a multiple of 32) the 32-env CTAs."""
    s = small_batch_envs()
    n = {"small-1": s - 1, "small": s, "small+1": s + 1}.get(N) or int(N)
    assert (n <= s) == (N not in ("small+1", "20011"))
    cnt = run_row("dense64", n, 8, params_of(max_v=3.0, min_v=1.0, max_step=30), kind="d27", T=24 if n < 10000 else 14,
                  age=(18, 30), seed=n, obs_every=1 if n < 10000 else 4)
    assert n < 8 or cnt["lose"] > 0
    assert n < 30 or (cnt["coll"] > 0 and cnt["restart"] > 0)


@pytest.mark.parametrize("city", CITIES)
def test_observe_after_set_state(city):
    """observe() (the DO_STEP = false instance) after set_state on every city: random positions, including points next to
    the box edges, and velocities including zero vectors with signed zeros (the cached heading follows V_vector)."""
    from uavrl_b200 import engine
    ecity, ocity = cities(city)
    K, N = 4, 333
    rng = np.random.default_rng(7)
    W, H = ocity.c.width, ocity.c.h
    params = params_of(max_v=3.0)
    sc = hand_pool(ocity, N, K, rng)
    env = engine.EnvBatch(ecity, engine.UavParams(**params), N, max_subgoals=K)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
    env.reset(0)
    ob = O.OracleBatch(ocity, O.UavParams(**params), N, K)
    ob.reset(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
    px = rng.uniform(-2, W + 2, N); py = rng.uniform(-2, W + 2, N); pz = rng.uniform(-1, H + 1, N)
    px[:20] = rng.choice([0.0, W, 19.5, W - 19.5, 20.0, W - 20.0], 20)          # the 75 planar probes reach +-20 m
    vx = rng.uniform(-3, 3, N); vy = rng.uniform(-3, 3, N)
    vx[20:40] = rng.choice([0.0, -0.0], 20); vy[20:40] = rng.choice([0.0, -0.0], 20)
    V = np.hypot(vx, vy)
    step = rng.integers(0, 150, N).astype(np.int32)
    env.set_state(px=px, py=py, pz=pz, vx=vx, vy=vy, V=V, step=step)
    for k, v in (("px", px), ("py", py), ("pz", pz), ("vx", vx), ("vy", vy), ("V", V), ("step", step)):
        getattr(ob, k)[:] = v
    got = env.observe().cpu().numpy()
    want = ob.state(want64=True)[1]
    assert_obs(got, want, city)
    assert (want[20:40, 7] > 3).any() and (want[20:40, 7] == 0).any()     # both directions of a zero V_vector
    env.close()


@pytest.mark.parametrize("city", ["empty", "one", "dense64", "box300x800", "apf"])
def test_device_pool_generator_equals_host_generator(city):
    """uavrl_env_generate_pool (device RRT) writes the same pool as uavrl_make_scenarios on the non-shipped cities:
    start, goal, sub-goals and n_sub bit for bit."""
    from uavrl_b200 import engine
    ecity, _ = cities(city)
    K, Pn = 64, 256
    a = engine.EnvBatch(ecity, engine.UavParams(**params_of(max_v=2.0)), 8, max_subgoals=K)
    b = engine.EnvBatch(ecity, engine.UavParams(**params_of(max_v=2.0)), 8, max_subgoals=K)
    sc = a.make_scenarios(Pn, seed=13)
    b.generate_pool(Pn, seed=13)
    pb = b.get_pool()
    for k in ("start", "goal", "sub", "n_sub"):
        assert np.array_equal(pb[k], sc[k]), k
    a.close(); b.close()


def test_threaten_rate_next_to_every_boundary():
    """threaten_rate (threat_kernel) on points 1 ulp either side of every R, H and box bound of the dense 64-cylinder city
    and of the 300 x 800 box, against OracleCity.threaten_rate."""
    from uavrl_b200 import engine
    rng = np.random.default_rng(3)
    for kind in ("dense64", "box300x800"):
        ecity, ocity = cities(kind)
        L, W, H, b = make_city(kind)
        pts = []
        up = lambda v: np.nextafter(v, np.inf)         # noqa: E731
        dn = lambda v: np.nextafter(v, -np.inf)        # noqa: E731
        for cx, cy, cz, R, Hc in b:
            for th in rng.uniform(0, 2 * np.pi, 4):
                for x in (cx + R * math.cos(th), up(cx + R * math.cos(th)), dn(cx + R * math.cos(th))):
                    pts.append((x, cy + R * math.sin(th), min(Hc, H) * 0.5))
            pts += [(cx + R, cy, 1.0), (up(cx + R), cy, 1.0), (dn(cx + R), cy, 1.0), (cx, dn(cy - R), 1.0)]
            pts += [(cx, cy, Hc), (cx, cy, up(Hc)), (cx, cy, dn(Hc))]
        for v in (0.0, -0.0, up(0.0), dn(0.0), W, up(W), dn(W), L, up(L)):
            pts += [(v, W / 2, 10.0), (W / 2, v, 10.0)]
        for v in (0.0, dn(0.0), H, up(H), dn(H)):
            pts.append((W / 3, 3.0, v))
        pts = np.array(pts)
        env = engine.EnvBatch(ecity, engine.UavParams(), 1, max_subgoals=4)
        got = env.threaten_rate(pts)
        want = ocity.threaten_rate(pts)
        assert np.array_equal(got, want), (kind, int((got != want).sum()))
        assert 0 < want.sum() < len(want)
        env.close()


@pytest.mark.parametrize("pset", [0, 1], ids=["steering_pi", "min_v_0"])
def test_kernel_matches_reference_off_the_shipped_parameters(pset):
    """The kernel on tests/golden/env_params_golden.npz (the unmodified reference UAV with overridden Max_V / Min_V /
    Steering_angle / Max_Step / climb on a generated city), all episodes of one parameter set in one batch, every action kind
    of the episode's mode.  Fails without the heading (steering_pi) and zero-velocity (min_v_0) fixes."""
    from uavrl_b200 import _lib, engine
    g = np.load(os.path.join(GOLDEN, "env_params_golden.npz"))
    d, p = g["dims"], g["params"][pset]
    city = engine.City(d[0], d[1], d[2], g["buildings"])
    params = engine.UavParams(p[0], p[1], p[2], p[4], int(p[3]))
    eps = [e for e in (episode(g, i) for i in range(int(g["epn_episodes"]))) if int(e["pset"]) == pset]
    checked = 0
    for mode in (0, 1):
        sel = [e for e in eps if int(e["mode"]) == mode]
        kinds = ("ACT_CONT_F64",) if mode == 0 else ("ACT_DISCRETE27",)
        for kname in kinds:
            n, K = len(sel), sel[0]["sub"].shape[0]
            env = engine.EnvBatch(city, params, n, max_subgoals=K, auto_reset=False)
            env.set_pool(np.stack([e["start"] for e in sel]), np.stack([e["goal"] for e in sel]), np.array([e["heading"] for e in sel]),
                         np.stack([e["sub"] for e in sel]), np.array([e["n_sub"] for e in sel]), np.array([e["alias0"] for e in sel]))
            env.reset(0)
            obs0 = env.observe().cpu().numpy()
            for i, e in enumerate(sel):
                assert_obs(obs0[i], e["obs0"], "obs0 ep%d" % i)
            for t in range(max(len(e["action"]) for e in sel)):
                if mode == 0:
                    act = torch.tensor([e["action"][t] if t < len(e["action"]) else 0.0 for e in sel], dtype=torch.float64, device="cuda")
                else:
                    act = torch.tensor([int(e["action"][t]) if t < len(e["action"]) else 13 for e in sel], dtype=torch.int32, device="cuda")
                o = {k: v.cpu().numpy() for k, v in env.step(act, kind=getattr(_lib, kname)).items()}
                st = env.get_state()
                for i, e in enumerate(sel):
                    if t >= len(e["action"]):
                        continue
                    w = "ep%d t%d" % (i, t)
                    assert (o["done"][i], o["info"][i], o["collision"][i]) == (e["done_ret"][t], e["info"][t], e["collision"][t]), w
                    assert (st["step"][i], st["cursor"][i], o["ended"][i]) == (e["step"][t], e["cursor"][t], e["done"][t]), w
                    assert_close64(st["reward64"][i], e["reward"][t], 1e-9, w + " reward")
                    for k in F64:
                        assert_close64(st[k][i], e[k][t], 1e-9, w + " " + k)
                    assert_obs(o["obs"][i], e["obs"][t], w)
                    checked += 1
            env.close()
    assert checked > 150
