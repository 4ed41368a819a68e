"""Moving obstacles (uavrl_env_set_motion): per-step time of env.step and of train_run iterations with the optional models off,
on without motion, with motion, and with motion and APF, on the shipped 26-cylinder city and on a 64-cylinder one.

python tools/bench_motion.py [--envs 4096 16384] [--steps 200] [--iters 100] [--rounds 3]

Configurations run alternately, `rounds` times each, and every number is the median over the rounds of CUDA-event time per
step (env.step) or per iteration (train_run, DDQN 100-64-64-27, one update per iteration).  "extras" turns on the episode
records, the lightest optional model, so that the step runs env_extras_kernel.  The card's name, power limit and maximum SM
clock are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else (torch.cuda.get_device_name(0), "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def city(nb):
    from uavrl_b200 import engine
    g = np.load(os.path.join(ROOT, "tests", "golden", "env_golden.npz"))
    b = g["buildings"]
    if nb > b.shape[0]:
        rng = np.random.default_rng(nb)
        extra = np.zeros((nb - b.shape[0], 5))
        extra[:, 0] = rng.uniform(0, g["dims"][0], len(extra)); extra[:, 1] = rng.uniform(0, g["dims"][1], len(extra))
        extra[:, 3] = rng.uniform(5, 20, len(extra)); extra[:, 4] = rng.uniform(10, 60, len(extra))
        b = np.concatenate([b, extra])
    p = g["uav_params"]
    vel = np.random.default_rng(7).normal(0, 1.5, (nb, 3))
    return engine.City(g["dims"][0], g["dims"][1], g["dims"][2], b), engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3])), vel


def make(cfg, N, nb):
    from uavrl_b200 import engine
    c, params, vel = city(nb)
    env = engine.EnvBatch(c, params, N, max_subgoals=64, auto_reset=True)
    env.generate_pool(max(N, 4096), seed=1)
    if cfg != "off":
        env.set_records(1)                                     # the extras step; every record beyond slot 0 is dropped
    if cfg == "motion_apf":
        env.set_extras(obstacle_v=vel)
    if cfg in ("motion", "motion_apf"):
        env.set_motion(vel)
    env.reset(0)
    return env


def time_events(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn(n)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n                          # microseconds per step / iteration


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 16384])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    cases = [(cfg, 26) for cfg in ("off", "extras", "motion", "motion_apf")] + [("motion", 64), ("off", 64)]
    res = {"card": card(), "step_us": {}, "train_iter_us": {}}
    for N in a.envs:
        acts = torch.randint(0, 27, (N,), dtype=torch.int32, device="cuda")
        built = {}
        for cfg, nb in cases:
            env = make(cfg, N, nb)
            L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=64, replay_capacity=8 * N, lockstep_envs=N)
            L.init_params(0)
            engine.train_run(env, L, 20, eps=0.2)              # warm-up: modules, the ring past batch_size
            for _ in range(10):
                env.step(acts)
            built[(cfg, nb)] = (env, L)
        st = {k: [] for k in built}; it = {k: [] for k in built}
        for _ in range(a.rounds):
            for k, (env, L) in built.items():
                st[k].append(time_events(lambda n: [env.step(acts) for _ in range(n)], a.steps))
                it[k].append(time_events(lambda n: engine.train_run(env, L, n, eps=0.2, want_stats=False), a.iters))
        for k in built:
            name = "%s_%dcyl_N%d" % (k[0], k[1], N)
            res["step_us"][name] = round(float(np.median(st[k])), 2)
            res["train_iter_us"][name] = round(float(np.median(it[k])), 2)
        del built
    print(json.dumps(res))


if __name__ == "__main__":
    main()
