"""Grouped SAC learners: G independent SAC trainers (the shipped shape: actor 100-64-{2,2}, critics 102-64-64-2, batch 64 each)
over one batch of 4096 envs in lockstep, for G in {1, 16, 256, 4096}.  One JSON line per G: iteration time (CUDA events over
the timed iterations, after warm-up), env steps/s, trainer updates/s, the device memory the learner holds, the time of one
federate_actors call (Federated_Learning_AC across the G actors), and the GPU's name, power limit and maximum SM clock read in
the same run.  bench.py stays the headline measurement.

    python tools/bench_sac_trainers.py [--envs 4096] [--trainers 1,16,256,4096] [--steps 500] [--warmup 50]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--trainers", default="1,16,256,4096")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--frames", type=int, default=128, help="replay ring frames (every trainer holds frames x envs/G transitions)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sac_trainers needs a CUDA device")
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    N, B = a.envs, a.batch
    info = gpu_info()
    for G in [int(x) for x in a.trainers.split(",")]:
        env = engine.EnvBatch(city, params, N, max_subgoals=64, device=0, auto_reset=True)
        sc = env.make_scenarios(2048, seed=42)
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        env.reset(0)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        L = engine.SacLearner(100, 64, 2, 1.0, 1e-4, 1e-3, 1e-4, 1.0, 0.99, 0.05, batch_size=B, replay_capacity=N * a.frames,
                              lockstep_envs=N, seed=1234, device=0, trainers=G)
        L.init_params(0)
        engine.sac_train_run(env, L, max(a.warmup, (B * G) // N + 2), want_stats=False)   # every trainer holds > B transitions
        torch.cuda.synchronize()
        footprint = free0 - torch.cuda.mem_get_info(0)[0]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        st = engine.sac_train_run(env, L, a.steps)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        assert st.updates == a.steps and torch.isfinite(torch.tensor(st.last_loss))
        fed = []
        for _ in range(6):                                   # first call warms up; median of the other five
            f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f0.record()
            L.federate_actors()
            f1.record()
            torch.cuda.synchronize()
            fed.append(f0.elapsed_time(f1))
        print(json.dumps({
            "trainers": G, "envs": N, "envs_per_trainer": N // G, "batch_per_trainer": B,
            "network": "SAC actor 100-64-{2,2}, critics 102-64-64-2",
            "iteration_us": ms * 1e3, "env_steps_per_s": N / (ms * 1e-3), "trainer_updates_per_s": G / (ms * 1e-3),
            "device_footprint_bytes": int(footprint), "federate_actors_us": sorted(fed[1:])[2] * 1e3,
            "timed_iterations": a.steps, "last_loss": float(st.last_loss), "gpu": info}), flush=True)
        L.close(); env.close()
        del L, env
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
