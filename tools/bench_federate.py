#!/usr/bin/env python
"""Selective federated aggregation (Learner.federate, PathPlan_City.Federated_Learning_choice) across G trainers of the
DQN 100-64-64-27 network on 4096 lockstep envs: milliseconds per call (device events around several calls after a
warm-up call, probes drawn from the ring) and the ratio to one episode of the plug-in's run_eposide loop at the same G
(lockstep iterations in chunks of 16 until as many episodes ended as there are envs).  One JSON line per G, with the
card's name, power limit and maximum SM clock read in the same run.

A call costs O(G^2): G (G - 1) 10 forward rows and, per round, an average over (G - 1) / 2 parameter vectors."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--trainers", default="16,256,1024,4096")
    ap.add_argument("--calls", type=int, default=3, help="timed federate() calls per G")
    ap.add_argument("--frames", type=int, default=32, help="replay ring frames")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_federate needs a CUDA device")
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    N, hidden = a.envs, [64, 64]
    info = gpu_info()
    for G in [int(x) for x in a.trainers.split(",")]:
        env = engine.EnvBatch(city, params, N, max_subgoals=64, device=0, auto_reset=True)
        sc = env.make_scenarios(2048, seed=42)
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        env.reset(0)
        L = engine.Learner(100, hidden, 27, False, engine.ALGO_DQN, lr=5e-4, gamma=0.99, batch_size=16, update_loop=3,
                           replay_capacity=N * a.frames, lockstep_envs=N, seed=1234, device=0, trainers=G)
        L.init_params(0)
        engine.train_run(env, L, max(16, (16 * G) // N + 2), 0.1, want_stats=False)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        # one episode of run_eposide: chunks of 16 lockstep iterations until N episodes ended
        ended, iters = 0, 0
        e0.record()
        while ended < N and iters < 64 * int(p[3]):
            ended += engine.train_run(env, L, 16, 0.1).episodes_ended
            iters += 16
        e1.record()
        torch.cuda.synchronize()
        episode_ms = e0.elapsed_time(e1)
        L.federate()                                                   # warm-up
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.calls):
            L.federate()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.calls
        P = L.P
        k = (G - 1) // 2
        print(json.dumps({
            "trainers": G, "envs": N, "network": "DQN 100-64-64-27", "params_per_trainer": P,
            "federate_ms": ms, "episode_ms": episode_ms, "episode_iterations": iters, "federate_over_episode": ms / episode_ms,
            "average_read_bytes": G * k * P * 4, "forward_rows": G * (G - 1) * 10, "timed_calls": a.calls,
            "gpu": info}), flush=True)
        L.close(); env.close()
        del L, env
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
