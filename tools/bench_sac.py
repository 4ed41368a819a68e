"""BASELINE configs[4]: SAC continuous (the trainer the reference ships) on 16 384 envs — env steps/s and updates/s.
Secondary measurement (bench.py stays on configs[1]).  python tools/bench_sac.py [--envs N] [--batch B] [--steps K] [--per 0|1]
[--profile].  --per 1: prioritised replay (SumTrees over the ring, weighted critic losses, the e_b write-back); --profile: per-kernel
device time over the timed steps from torch.profiler instead of the end-to-end rate."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--replay", type=int, default=1 << 20)
    ap.add_argument("--per", type=int, choices=(0, 1), default=0)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    B = a.batch or a.envs
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import _lib, engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    env = engine.EnvBatch(city, params, a.envs, max_subgoals=64, device=0, auto_reset=True)
    sc = env.make_scenarios(2048, seed=42)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    env.reset(0)
    L = engine.SacLearner(100, 64, 2, 1.0, 1e-4, 1e-3, 1e-4, 1.0, 0.99, 0.05, batch_size=B, replay_capacity=a.replay,
                          lockstep_envs=a.envs, seed=7, device=0)
    L.init_params(0)
    if a.per:
        L.per_enable()
    frames = (a.replay + a.envs - 1) // a.envs + 1
    engine.sac_train_run(env, L, frames, False, want_stats=False)          # prefill the ring (> L2)
    engine.sac_train_run(env, L, 10, True, want_stats=False)
    torch.cuda.synchronize()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            engine.sac_train_run(env, L, a.steps, True, want_stats=False)
            torch.cuda.synchronize()
        us = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                us[ev.name] = us.get(ev.name, 0.0) + ev.device_time
        print(json.dumps({"per": a.per, "steps": a.steps, "gpu": torch.cuda.get_device_name(0),
                          "kernel_us_per_step": {k.split("(")[0][-80:]: v / a.steps for k, v in sorted(us.items(), key=lambda kv: -kv[1])}}),
              flush=True)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = _lib.launch_count()
    e0.record()
    st = engine.sac_train_run(env, L, a.steps, True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    sc_ = L.scalars()
    print(json.dumps({"metric": "env steps/sec (+ SAC updates/sec), 500x500x100 city", "value": a.envs * a.steps / (ms * 1e-3),
                      "unit": "env_steps/s", "updates_per_s": a.steps / (ms * 1e-3), "ms_per_step": ms / a.steps, "n_gpus": 1,
                      "steps": a.steps, "gpu_launches": int(_lib.launch_count() - n0), "per": a.per,
                      "gpu": torch.cuda.get_device_name(0),
                      "config": {"workload": "%d envs, continuous update_PathPlan, SAC actor 100-64-(2,2) + 2 critics 102-64-64-2, "
                                             "batch %d, replay %d (> L2), 1 update / lockstep iteration" % (a.envs, B, a.replay)},
                      "episodes_ended": int(st.episodes_ended), "last_loss": float(st.last_loss), "log_alpha": sc_["log_alpha"]},
                     default=float), flush=True)
    assert np.isfinite(st.last_loss)


if __name__ == "__main__":
    main()
