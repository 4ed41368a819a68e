#!/usr/bin/env python
"""Golden episodes of moving obstacles: the reference's scene-change hook PathPlan_City.run() made live.

The reference calls PathPlan_City.run() ("scene elements change", Envs/PathPlan_City.py:424,442) at the top of every lockstep
iteration, before any UAV observes or moves; it and every obstacle's run() are `pass` as shipped.  Here every building of the
shipped 26-cylinder city is given the `v` attribute cal_force reads and a run() that applies the port's rule (include/uavrl.h,
uavrl_env_set_motion) with the reference's Loc arithmetic:
    position += Loc(vx, vy, 0); then x reflected once at 0 / len (vx reversed), y at 0 / width (vy reversed)
and env.run() calls each building's run().  The UNMODIFIED reference UAV is then driven in the reference's own loop order:
run(), state_test = uav.state(), action, Move_Agent.  Three configurations: continuous actions with APF off, with APF on
(some obstacles still, one with vz != 0), and the discrete-27 route (make_golden.UAV27, APF off: its step has no APF branch).
The table is carried across the episodes of a configuration, as the reference carries it across resets.

Run in the build container only (needs the reference):   python tests/golden/make_motion_golden.py
Writes tests/golden/motion_golden.npz with, per episode (prefix cfg<c>_ep<i>_): the scenario (start, goal, heading, sub,
n_sub, alias0); the table ([n][4] = x, y, vx, vy) before the episode's first run() (`tab0`) and after it (`tab1`); per
iteration the table after run() as `tab_digest` (motion_oracle.table_digest: BLAKE2b of its fp64 bytes, so it pins every bit
without storing ~20 KB of incompressible centres per step) and `vsign` (the velocity sign bits, which show the reflections),
`state_test`, Move_Agent's `next_state`, action, reward, done_ret, info, collision and position; with APF (whose force shifts
the queue every step) the remaining sub-goal queue (`subq`, zero padded)."""
import copy
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (loads the reference through oracle/ref_harness; seeds everything with 42)
from BaseClass.CalMod import Loc  # noqa: E402  (reference)

sys.path.insert(0, os.path.dirname(HERE))
from motion_oracle import table_digest, velocity_signs  # noqa: E402


def obstacle_run(self):
    """The port's run() for one obstacle, in Loc arithmetic; self.env_len / env_width are the city box."""
    p = self.position + Loc(self.v.x, self.v.y, 0)
    if p.x < 0:
        p.x = -p.x
        self.v.x = -self.v.x
    elif p.x > self.env_len:
        p.x = self.env_len - (p.x - self.env_len)
        self.v.x = -self.v.x
    if p.y < 0:
        p.y = -p.y
        self.v.y = -self.v.y
    elif p.y > self.env_width:
        p.y = self.env_width - (p.y - self.env_width)
        self.v.y = -self.v.y
    self.position = Loc(p.x, p.y, self.position.z)


def table(env):
    return np.array([[t.position.x, t.position.y, t.v.x, t.v.y] for t in env.buildings], np.float64)


def main():
    s = mg.sim_mod.simulator()
    env = s.env
    uav = env.Agents[0]
    rng = np.random.default_rng(20261018)
    nb = len(env.buildings)
    pos0 = [copy.copy(t.position) for t in env.buildings]
    vel = np.zeros((nb, 3))
    ang = rng.uniform(0, 2 * np.pi, nb)
    spd = rng.uniform(1.0, 4.0, nb)
    vel[:, 0] = spd * np.cos(ang)
    vel[:, 1] = spd * np.sin(ang)
    vel[np.arange(nb) % 5 == 3] = 0.0                           # still obstacles: no force, no motion
    vel[4, 2] = 0.5                                             # a vertical component: only |v| sees it
    for t in env.buildings:
        t.env_len, t.env_width = float(env.len), float(env.width)
        t.run = types.MethodType(obstacle_run, t)
    env.run = lambda: [t.run() for t in env.buildings]
    u27 = mg.UAV27(copy.copy(uav.param), env)
    out = {"obstacle_v": vel, "buildings": np.array([[t.position.x, t.position.y, t.position.z, t._R, t._H] for t in env.buildings]),
           "dims": np.array([env.len, env.width, env.h], np.float64),
           "uav_params": np.array([uav.Max_V, float(uav.param.get("Min_V")), uav.Steering_angle, uav.Max_Step], np.float64),
           "climb_rate": np.float64(mg.UAV27.climb_rate)}
    walls = np.zeros(4, np.int64)                               # reflections seen at x = 0, x = len, y = 0, y = width
    total = 0
    cfgs = (("cont", 0, uav), ("apf", 1, uav), ("d27", 0, u27))
    out["n_cfg"] = np.int32(len(cfgs))
    for c, (name, apf, agent) in enumerate(cfgs):
        for t, p, v in zip(env.buildings, pos0, vel):           # every configuration starts from the XML table
            t.position = copy.copy(p)
            t.v = Loc(float(v[0]), float(v[1]), float(v[2]))
        env.Agents[0] = agent
        agent.APF_Enabled = apf
        eps = []
        for i in range(3):
            env.Scene_Random_Reset()
            nsub = len(agent.sub_goals)
            sub = np.zeros((mg.KMAX, 3))
            for k, sg in enumerate(agent.sub_goals):
                sub[k] = (sg.x, sg.y, sg.z)
            ep = dict(start=np.array([agent.position.x, agent.position.y, agent.position.z]),
                      goal=np.array([agent.goal.x, agent.goal.y, agent.goal.z]), heading=np.float64(agent.V_dir),
                      sub=sub, n_sub=np.int32(nsub), alias0=np.uint8(int(agent.sub_goals[0] is agent.position)))
            ep["tab0"] = table(env)
            rec = {k: [] for k in ("tab_digest", "vsign", "state_test", "next_state", "action", "reward", "done_ret", "info",
                                   "collision", "px", "py", "pz", "subq")}
            for _ in range(200):
                if agent.done:
                    break
                tb = table(env)
                env.run()                                       # PathPlan_City.run(): every obstacle moves
                ta = table(env)
                walls += [int(np.sum((tb[:, 2] < 0) & (ta[:, 2] > 0))),
                          int(np.sum((tb[:, 2] > 0) & (ta[:, 2] < 0))), int(np.sum((tb[:, 3] < 0) & (ta[:, 3] > 0))),
                          int(np.sum((tb[:, 3] > 0) & (ta[:, 3] < 0)))]
                state_test = np.asarray(agent.state(), np.float64)
                before = (agent.position.x, agent.position.y, agent.position.z)
                if name == "d27":
                    act = float(rng.integers(0, 27)) if i == 0 else float(rng.integers(0, 3) * 9 + rng.integers(0, 3) * 3 + 2)
                    reward, done, info = agent.update_PathPlan27(int(act))
                    next_state = agent.state()
                else:
                    act = rng.uniform(-1, 1) if i == 1 else mg.seek_action(agent, rng.normal(0, 0.25))
                    next_state, reward, done, info = env.Move_Agent(0, [act, rng.uniform(-1, 1)])
                q = np.zeros((mg.KMAX, 3))
                for k, sg in enumerate(agent.sub_goals):
                    q[k] = (sg.x, sg.y, sg.z)
                if not rec["tab_digest"]:
                    ep["tab1"] = ta
                for k, v in (("tab_digest", np.frombuffer(table_digest(ta), np.uint8)), ("vsign", velocity_signs(ta)),
                             ("state_test", state_test),
                             ("next_state", np.asarray(next_state, np.float64)), ("action", act), ("reward", reward),
                             ("done_ret", int(done)), ("info", mg.INFO[info]),
                             ("collision", int((agent.position.x, agent.position.y, agent.position.z) == before)),
                             ("px", agent.position.x), ("py", agent.position.y), ("pz", agent.position.z), ("subq", q)):
                    rec[k].append(v)
            if not apf:
                del rec["subq"]
            for k, v in rec.items():
                dt = np.uint8 if k in ("done_ret", "info", "collision", "tab_digest", "vsign") else np.float64
                ep[k] = np.asarray(v, dt)
            eps.append(ep)
            total += len(ep["action"])
            print("%s episode %d: %d steps, %d collisions, final info %d" % (name, i, len(ep["action"]), int(ep["collision"].sum()),
                                                                            int(ep["info"][-1])))
        mg.pack_episodes(eps, "cfg%d_ep" % c, out)
    env.Agents[0] = uav
    print("motion_golden.npz: %d steps, reflections at x=0 / x=len / y=0 / y=width: %s" % (total, walls.tolist()))
    assert (walls > 0).all(), "every wall must reflect some obstacle"
    np.savez_compressed(os.path.join(HERE, "motion_golden.npz"), **out)


if __name__ == "__main__":
    main()
