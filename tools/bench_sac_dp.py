"""Data-parallel SAC: time per lockstep iteration and the bytes an update exchanges.  Prints one JSON line.

    python tools/bench_sac_dp.py [--envs N] [--batch B] [--steps K] [--reps R]
        world = 1 (BASELINE configs[4] size: 16 384 envs, batch 16 384): sac_train_run against sac_train_run_dp after
        connect_self (the fused exchanges on the local buffer), alternated R times in one process.
    torchrun --nproc-per-node W tools/bench_sac_dp.py ...
        W ranks, each with its own env shard and ring: the fused update_replay_dp loop against the split form with NCCL
        all-reduces between the phases, alternated.

The card's name, power limit and maximum SM clock are read in the same run; every time is one measured on that card."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def exchange_bytes(Pa, Pc):
    """8-byte words one rank pushes to each peer per update: both critics' gradients + 2 sums, the actor's gradient + 2 sums."""
    return 8 * ((2 * Pc + 2) + (Pa + 2))


def card(dev):
    q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else (torch.cuda.get_device_name(dev), "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--replay", type=int, default=1 << 20)
    a = ap.parse_args()
    B = a.batch or a.envs
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(dev)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))

    def pair():
        env = engine.EnvBatch(city, params, a.envs, max_subgoals=64, device=dev, auto_reset=True)
        sc = env.make_scenarios(2048, seed=42 + rank)
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        env.reset(0)
        S = engine.SacLearner(100, 64, 2, 1.0, 1e-4, 1e-3, 1e-4, 1.0, 0.99, 0.05, batch_size=B, replay_capacity=a.replay,
                              lockstep_envs=a.envs, seed=7 + rank, device=dev)
        S.init_params(0)
        engine.sac_train_run(env, S, (a.replay + a.envs - 1) // a.envs + 1, False, want_stats=False)     # ring > L2
        return env, S

    (env_a, A), (env_b, Bl) = pair(), pair()
    if world > 1:
        Bl.connect_peers(dist, rank, world)
        xs = (A.exchange_tensor(0), A.exchange_tensor(1))

        def run_a(k):                           # split form, NCCL between the phases
            for _ in range(k):
                engine.sac_train_run(env_a, A, 1, False, want_stats=False)
                A.critic_grads(B * world)
                dist.all_reduce(xs[0], op=dist.ReduceOp.SUM)
                A.apply_critic_grads()
                A.actor_grads()
                dist.all_reduce(xs[1], op=dist.ReduceOp.SUM)
                A.apply_actor_grads()
        names = ("nccl_split", "fused")
    else:
        Bl.connect_self()

        def run_a(k):
            engine.sac_train_run(env_a, A, k, True, want_stats=False)
        names = ("plain", "fused_self")

    def run_b(k):
        engine.sac_train_run_dp(env_b, Bl, k, B * world)

    times = {n: [] for n in names}
    for fn in (run_a, run_b):
        fn(10)                                  # warm-up of every shape the timed windows use
    for _ in range(a.reps):
        for n, fn in zip(names, (run_a, run_b)):
            if dist:
                dist.barrier(device_ids=[dev])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(a.steps)
            e1.record()
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1)], device="cuda", dtype=torch.float64)
            if dist:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            times[n].append(1e3 * float(ms) / a.steps)
    Pa, Pc = A.P[0], A.P[1]
    out = {"metric": "us per lockstep iteration (1 SAC update each)", "world": world, "envs_per_rank": a.envs, "batch_per_rank": B,
           "steps": a.steps, "reps": a.reps, "actor_params": Pa, "critic_params": Pc,
           "exchange_bytes_per_update_per_peer": exchange_bytes(Pa, Pc),
           "us_per_iter": {n: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for n, v in times.items()}}
    out.update(card(dev))
    if rank == 0:
        print(json.dumps(out), flush=True)
    for x in (A, Bl, env_a, env_b):
        x.close()
    if dist:
        dist.barrier(device_ids=[dev])
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
