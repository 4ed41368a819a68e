"""Grouped learners: G independent DQN trainers (100-64-64-27, batch 64 each, the reference's Batch_Size) over one batch of
4096 envs in lockstep, for G in {1, 16, 256, 4096}.  One JSON line per G: iteration time (CUDA events over the timed
iterations, after warm-up), env steps/s, trainer updates/s, the weight-image bytes the kernels stage into shared memory per
iteration (computed from the shapes) and that traffic over time as a share of the H100 SXM's 3.35 TB/s, the per-kernel split
of one iteration, and the GPU's name and power limit read in the same run.  bench.py stays the headline measurement.
--per gives every trainer its own prioritised replay (uavrl_per_enable_trainers); the line then carries "prioritised_replay".

    python tools/bench_trainers.py [--envs 4096] [--trainers 1,16,256,4096] [--steps 2000] [--warmup 200] [--per]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def rup(x, m):
    return -(-x // m) * m


def image_bytes(in_dim, hidden, n_actions):
    """Tensor-core weight images (tc_build in csrc/tc_forward.cu): the forward image (hi|lo blocks + biases) and the training
    image (forward image + transposed hi|lo blocks of layers >= 1)."""
    widths = list(hidden) + [n_actions]
    k, off, bias, t = rup(in_dim, 8), 0, 0, 0
    for i, w in enumerate(widths):
        n = 32 if i == len(widths) - 1 else rup(w, 16)
        off += 2 * n * k * 4
        bias += n
        if i > 0:
            t += 2 * k * n * 4
        k = n
    fwd = rup(off + 4 * bias, 16)
    return fwd, rup(fwd + t, 16)


def staged_bytes(L, N, G, B, algo_dqn, fwd, train):
    """Bytes one lockstep iteration copies from global into shared memory as weight images: every CTA of the act pass stages
    the forward image once; every training CTA stages the training image and, for the TD targets, the forward image of each
    network it evaluates (fused: inside the training kernel; else in the stand-alone TD passes)."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    Ng = N // G
    r_act, r_td = L.route(Ng), L.route(B)
    act_ctas = min(-(-Ng // r_act["fwd_rows"]), n_sm)
    train_ctas = min(-(-B // r_td["train_rows"]), n_sm)
    n_td = 1 if algo_dqn else 2
    if r_td["td_fused"]:
        per_update = train_ctas * (train + n_td * fwd)
    else:
        td_ctas = min(-(-B // r_td["fwd_rows"]), n_sm)
        per_update = train_ctas * train + n_td * td_ctas * fwd
    return G * (act_ctas * fwd + per_update)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--trainers", default="1,16,256,4096")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--frames", type=int, default=128, help="replay ring frames (every trainer holds frames x envs/G transitions)")
    ap.add_argument("--per", action="store_true", help="prioritised replay, one SumTree per trainer")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trainers needs a CUDA device")
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import _lib, engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    N, B, hidden = a.envs, a.batch, [64, 64]
    fwd, train = image_bytes(100, hidden, 27)
    info = gpu_info()
    for G in [int(x) for x in a.trainers.split(",")]:
        env = engine.EnvBatch(city, params, N, max_subgoals=64, device=0, auto_reset=True)
        sc = env.make_scenarios(2048, seed=42)
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        env.reset(0)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        L = engine.Learner(100, hidden, 27, False, engine.ALGO_DQN, lr=5e-4, gamma=0.99, batch_size=B, update_loop=3,
                           replay_capacity=N * a.frames, lockstep_envs=N, seed=1234, device=0, trainers=G)
        L.init_params(0)
        if a.per:
            L.per_enable_trainers()
        engine.train_run(env, L, max(a.warmup, (B * G) // N + 2), 0.1, want_stats=False)   # every trainer holds > B transitions
        torch.cuda.synchronize()
        footprint = free0 - torch.cuda.mem_get_info(0)[0]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        st = engine.train_run(env, L, a.steps, 0.1)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        assert st.updates == a.steps and torch.isfinite(torch.tensor(st.last_loss))
        prof = engine.train_profile(env, L, 200, 0.1) / 200           # event-separated kernels: a split, not a throughput
        sb = staged_bytes(L, N, G, B, True, fwd, train)
        extra = {"prioritised_replay": True} if a.per else {}
        print(json.dumps({
            "trainers": G, "envs": N, "envs_per_trainer": N // G, "batch_per_trainer": B, "network": "DQN 100-64-64-27",
            "iteration_us": ms * 1e3, "env_steps_per_s": N / (ms * 1e-3), "trainer_updates_per_s": G / (ms * 1e-3),
            "staged_image_bytes_per_iter": sb, "staged_image_GB_per_s": sb / (ms * 1e-3) / 1e9,
            "staged_share_of_3.35TBps": sb / (ms * 1e-3) / HBM_BYTES_PER_S,
            "profile_us": dict(zip(("act", "env_step", "td_target", "train", "weight_grad", "optimiser"), (float(x) * 1e3 for x in prof))),
            "device_footprint_bytes": int(footprint), "timed_iterations": a.steps, "last_loss": float(st.last_loss),
            "gpu": info, "launches": int(_lib.launch_count()), **extra}), flush=True)
        L.close(); env.close()
        del L, env
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
