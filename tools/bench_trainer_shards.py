"""Trainer groups sharded over the GPUs of one box: global G trainers over 4096 global envs in lockstep, rank r holding envs
[r N / W, (r + 1) N / W) and trainers [r G / W, (r + 1) G / W), for the DQN 100-64-64-27 network and for SAC (the shipped
shape), G in {256, 4096}.  One JSON line per configuration, printed by rank 0: iteration time (CUDA events over the timed
iterations after warm-up, the slowest rank), global trainer updates/s, and the device time of one aggregation call
(Learner.federate_sharded / SacLearner.federate_actors_sharded, after one warm-up call, the slowest rank), beside the card's
name, power limit and maximum SM clock read in the same run.

    torchrun --nproc-per-node W tools/bench_trainer_shards.py [--envs 4096] [--trainers 256,4096] [--steps 500] [--warmup 50]
    python tools/bench_trainer_shards.py ...                   (W = 1)"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


class _OneRank:
    """torch.distributed's all-gather for a world of one rank (no process group)."""

    @staticmethod
    def all_gather_into_tensor(out, inp):
        out.copy_(inp)


def gpu_info(dev):
    r = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--trainers", default="256,4096")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--frames", type=int, default=128, help="replay ring frames (every trainer holds frames x envs/G transitions)")
    ap.add_argument("--nets", default="dqn,sac")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trainer_shards needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(dev)
    dist = _OneRank
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    N, B = a.envs, a.batch
    NL = N // world
    info = gpu_info(dev)

    def slowest(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for net in a.nets.split(","):
        for G in [int(x) for x in a.trainers.split(",")]:
            GL = G // world
            env = engine.EnvBatch(city, params, NL, max_subgoals=64, device=dev, auto_reset=True)
            sc = env.make_scenarios(2048, seed=42)
            env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
            env.set_reset_stride(N)
            env.reset(rank * NL)
            if net == "dqn":
                L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DQN, lr=5e-4, gamma=0.99, batch_size=B, update_loop=3,
                                   replay_capacity=NL * a.frames, lockstep_envs=NL, seed=1234 + rank * GL, device=dev, trainers=GL)
                run = lambda n: engine.train_run(env, L, n, 0.1, want_stats=False)  # noqa: E731
                agg = lambda: L.federate_sharded(dist)  # noqa: E731
                name = "DQN 100-64-64-27"
            else:
                L = engine.SacLearner(100, 64, 2, 1.0, 1e-4, 1e-3, 1e-4, 1.0, 0.99, 0.05, batch_size=B, replay_capacity=NL * a.frames,
                                      lockstep_envs=NL, seed=1234 + rank * GL, device=dev, trainers=GL)
                run = lambda n: engine.sac_train_run(env, L, n, want_stats=False)  # noqa: E731
                agg = lambda: L.federate_actors_sharded(dist)  # noqa: E731
                name = "SAC actor 100-64-{2,2}, critics 102-64-64-2"
            L.init_params(rank * GL)
            L.fed_shard(rank, world)
            run(max(a.warmup, (B * G) // N + 2))                     # every trainer holds > B transitions
            torch.cuda.synchronize()
            ms, _ = timed(lambda: run(a.steps))
            ms = slowest(ms) / a.steps
            agg()                                                    # warm-up call
            torch.cuda.synchronize()
            agg_ms = slowest(timed(agg)[0])
            if rank == 0:
                print(json.dumps({
                    "network": name, "world": world, "trainers": G, "trainers_per_rank": GL, "envs": N, "envs_per_rank": NL,
                    "batch_per_trainer": B, "iteration_us": ms * 1e3, "trainer_updates_per_s": G / (ms * 1e-3),
                    "aggregation_ms": agg_ms, "timed_iterations": a.steps, "gpu": info}), flush=True)
            L.close(); env.close()
    if world > 1:
        dist.barrier(device_ids=[dev])
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
