#!/usr/bin/env python
"""Golden episodes of the reference UAV off the shipped UAV parameters and city.

env_golden.npz / env27_golden.npz pin the step at the shipped values only (Max_V 1, Min_V 0.6, Steering_angle 30 deg,
Max_Step 150, climb 1, the 26-cylinder 500 x 500 x 100 city).  Here the UNMODIFIED reference UAV (continuous actions through
env.Move_Agent -> UAV.update_PathPlan, discrete-27 through make_golden.UAV27) is driven with its `param` fields overridden on a
generated city: 24 cylinders with non-zero base z, some straddling the box edge, some taller than the box, in a
360 x 420 x 60 box (length != width: PathPlan_City.py:218 tests x and y against `width`).  Two parameter sets:

  set 0  Max_V 3, Min_V 1, Steering_angle pi, Max_Step 40, climb 2: continuous actions in [-3, 3], so |a0 * steering|
         reaches 3 pi and the heading leaves [0, 2 pi) after one wrap; discrete-27 at the same values.
  set 1  Max_V 2, Min_V 0, Steering_angle pi / 2, Max_Step 25, climb 0.5: discrete-27 with speed level 0 on half the steps,
         so V_vector = 0 * (cos, sin) carries signed zeros and calculate_angle of it is atan2(+-0, -0) = +-pi or
         atan2(+-0, +0) = +-0; continuous actions in [-1, 1] at the same values.

Episodes are set up by hand (UAV.reset's draws and an RRT-like straight path of 2-6 sub-goals, sub_goals[0] aliasing the
position in half of them), since RRT's start / goal regions are fixed to the shipped box.  Each records what
make_golden.record_episode records, plus `pset` (row of `params`) and `mode` (0 continuous, 1 discrete-27).

Run in the build container only (needs /root/reference):   python tests/golden/make_env_params_golden.py
"""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (loads the reference through oracle/ref_harness; seeds everything with 42)
from BaseClass.CalMod import Loc  # noqa: E402  (reference)
from Obstacles.building import building  # noqa: E402  (reference)

KMAX = 8
DIMS = (360.0, 420.0, 60.0)
# max_v, min_v, steering, max_step, climb_rate
PARAMS = np.array([[3.0, 1.0, math.pi, 40, 2.0],
                   [2.0, 0.0, math.pi / 2, 25, 0.5]], np.float64)


def make_city(rng, n=24):
    L, W, H = DIMS
    b = np.zeros((n, 5))
    b[:, 0] = rng.uniform(-10, W + 10, n)          # x is tested against width too
    b[:, 1] = rng.uniform(-10, W + 10, n)
    b[:, 2] = rng.uniform(0.5, 6.0, n)             # base z: only ever subtracted from itself
    b[:, 3] = rng.uniform(6, 30, n)
    b[:, 4] = rng.uniform(8, 90, n)                # some above h
    b[0, :2] = (-5.0, 200.0); b[1, :2] = (200.0, W + 4.0)          # straddling the box edge
    b[2, 4] = 3.0                                                  # below most flight heights
    return b


def set_params(u, p):
    u.Max_V, u.Steering_angle, u.Max_Step = float(p[0]), float(p[2]), int(p[3])
    u.param["Min_V"] = float(p[1])
    u.climb_rate = float(p[4])


def free_point(env, rng, lo, hi):
    while True:
        q = rng.uniform(lo, hi)
        if env.Threaten_rate(Loc(*q)) == 0:
            return q


def set_episode(env, u, rng, alias):
    """UAV.reset (Agents/UAV.py:335-366) with hand-made start, goal and sub-goal path."""
    L, W, H = DIMS
    start = free_point(env, rng, (5, 5, 5), (W - 5, W - 5, H - 10))
    goal = free_point(env, rng, (5, 5, 0), (W - 5, W - 5, H - 10))
    n_mid = int(rng.integers(0, 5))
    mids = [start + (goal - start) * (k + 1) / (n_mid + 1) + rng.normal(0, 4, 3) * (1, 1, 0.3) for k in range(n_mid)]
    first = start if alias else start + rng.normal(0, 3, 3) * (1, 1, 0)
    pts = [first] + mids + [goal]
    heading = rng.uniform(0, 2 * math.pi)
    u.Step = 0; u.score = 0; u.done = False; u.path = []; u.V_record = []; u.R_record = []
    u.V_vector = Loc(0, 0, 0)
    u.V_vector.x = u.Max_V * math.cos(heading)
    u.V_vector.y = u.Max_V * math.sin(heading)
    u.V = u.Calc_V()
    u.position = Loc(*start)
    u.goal = Loc(*goal)
    u.sub_goals = [u.position if (alias and i == 0) else Loc(*p) for i, p in enumerate(pts)]
    u.total_score = 0; u.path_len = 0
    sub = np.zeros((KMAX, 3))
    sub[:len(pts)] = pts
    return dict(start=np.array(start, np.float64), goal=np.array(goal, np.float64), heading=np.float64(heading),
                vx0=np.float64(u.V_vector.x), vy0=np.float64(u.V_vector.y), V0=np.float64(u.V), sub=sub,
                n_sub=np.int32(len(pts)), alias0=np.uint8(alias), obs0=u.state().astype(np.float64))


def record(env, u, ep, step_fn, sampler, rng, max_steps=200):
    keys = ("action", "reward", "done_ret", "info", "collision", "px", "py", "pz", "vx", "vy", "V",
            "step", "cursor", "done", "score", "total_score", "path_len")
    rec = {k: [] for k in keys}
    obs = []
    nsub = int(ep["n_sub"])
    # the step's own threat test (UAV.py:425, its only Threaten_rate call with APF off) is the collision flag: with speed 0
    # the position also stays put without one, so "position unchanged" (make_golden.record_episode) would not do here
    threat = env.Threaten_rate
    calls = []
    for _ in range(max_steps):
        if u.done:
            break
        act = sampler(u, rng)
        calls.clear()
        env.Threaten_rate = lambda p: calls.append(threat(p)) or calls[-1]
        try:
            reward, done, info = step_fn(act)
        finally:
            env.Threaten_rate = threat
        assert len(calls) in (1, 81)              # + the 80 probes of state() inside Move_Agent
        s = mg.snapshot(u)
        rec["action"].append(act); rec["reward"].append(reward); rec["done_ret"].append(int(done))
        rec["info"].append(mg.INFO[info])
        rec["collision"].append(int(calls[0]))
        for k in ("px", "py", "pz", "vx", "vy", "V", "step", "done", "score", "total_score", "path_len"):
            rec[k].append(s[k])
        rec["cursor"].append(nsub - s["nleft"])
        obs.append(np.asarray(u.state(), np.float64))
    for k in keys:
        dt = np.uint8 if k in ("done_ret", "info", "collision", "done") else np.int32 if k in ("step", "cursor") else np.float64
        ep[k] = np.asarray(rec[k], dt)
    ep["obs"] = np.stack(obs)
    return ep


def main():
    s = mg.sim_mod.simulator()
    env = s.env
    uav = env.Agents[0]
    rng = np.random.default_rng(20261016)
    b = make_city(rng)
    env.len, env.width, env.h = int(DIMS[0]), DIMS[1], DIMS[2]
    env.buildings = [building({"position": {"x": str(r[0]), "y": str(r[1]), "z": str(r[2])}, "_R": str(r[3]),
                               "_H": str(r[4]), "type": "building"}) for r in b]
    u27 = mg.UAV27(dict(uav.param), env)

    def cont_step(a):
        _, r, d, i = env.Move_Agent(0, [a, 0.0])
        return r, d, i

    def cont_sampler(bound):
        def f(u, g):
            if g.uniform() < 0.5:
                return float(g.uniform(-bound, bound))
            return mg.seek_action(u, g.normal(0, 0.25))
        return f

    def d27_sampler(p_slow):
        def f(u, g):
            i = int(np.clip(round(mg.seek_action(u, g.normal(0, 0.4))), -1, 1)) + 1 if g.uniform() < 0.6 else int(g.integers(0, 3))
            j = int(g.integers(0, 3))
            lv = 0 if g.uniform() < p_slow else int(g.integers(0, 3))
            return i * 9 + j * 3 + lv
        return f

    out = {"buildings": b, "dims": np.array(DIMS), "params": PARAMS}
    plan = [(0, 0, cont_sampler(3.0), 4), (0, 1, d27_sampler(0.2), 2),
            (1, 1, d27_sampler(0.5), 4), (1, 0, cont_sampler(1.0), 2)]
    eps = []
    for pset, mode, sampler, n in plan:
        for k in range(n):
            u = uav if mode == 0 else u27
            set_params(u, PARAMS[pset])
            env.Agents[0] = u
            ep = set_episode(env, u, rng, alias=(k % 2 == 0))
            ep = record(env, u, ep, cont_step if mode == 0 else u27.update_PathPlan27, sampler, rng)
            ep["pset"] = np.int32(pset); ep["mode"] = np.int32(mode)
            eps.append(ep)
            print("set %d mode %d: %3d steps, %d sub-goals, %2d collisions, pops %d, final info %d, obs[7] range [%.3f, %.3f], "
                  "V = 0 on %d steps" % (pset, mode, len(ep["action"]), int(ep["n_sub"]), int(ep["collision"].sum()),
                                         int(ep["cursor"][-1]), int(ep["info"][-1]), ep["obs"][:, 7].min(), ep["obs"][:, 7].max(),
                                         int((ep["V"] == 0).sum())))
    env.Agents[0] = uav
    mg.pack_episodes(eps, "ep", out)
    np.savez_compressed(os.path.join(HERE, "env_params_golden.npz"), **out)
    print("env_params_golden.npz: %d episodes, %d steps, %d KiB" % (len(eps), sum(len(e["action"]) for e in eps),
                                                                     os.path.getsize(os.path.join(HERE, "env_params_golden.npz")) // 1024))


if __name__ == "__main__":
    main()
