"""Policy evaluation on the device (engine.eval_run / engine.sac_eval_run): episodes/s, env steps/s and microseconds per
iteration over a held-out suite, next to the training loop's act + env-step cost at the same shape.

python tools/bench_eval.py [--envs 4096] [--episodes 16384] [--pool 16384]

DQN 100-64-64-27: the evaluation beside train_profile's act and env-step split of uavrl_train_run at the same env count.
SAC (the shipped 100-64 actor): beside sac_train_run with do_update = 0 (act + env step + ring commit), which has no
profile entry point.  Untrained networks rarely reach a goal, so episodes mostly end by max_step: the rates are those of
full-length episodes.  The card's name, power limit and maximum SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().split(",")) if q.returncode == 0 else (torch.cuda.get_device_name(0), "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--episodes", type=int, default=16384)
    ap.add_argument("--pool", type=int, default=16384)
    ap.add_argument("--train-iters", type=int, default=200)
    a = ap.parse_args()
    import uavrl_b200  # noqa: F401
    from uavrl_b200 import engine
    from bench import load_city
    dims, b, p = load_city()
    city = engine.City(dims[0], dims[1], dims[2], b)
    params = engine.UavParams(p[0], p[1], p[2], 1.0, int(p[3]))
    N = a.envs

    def env_with_pool(auto_reset):
        env = engine.EnvBatch(city, params, N, max_subgoals=64, device=0, auto_reset=auto_reset)
        env.generate_pool(a.pool, seed=43)
        return env

    out = {"envs": N, "episodes": a.episodes, **card()}
    ev = env_with_pool(False)
    for kind in ("dqn", "sac"):
        if kind == "dqn":
            L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DQN, batch_size=N, replay_capacity=1 << 20, lockstep_envs=N, seed=7)
            L.init_params(0)
            run = lambda: engine.eval_run(ev, L, a.episodes)  # noqa: E731
        else:
            L = engine.SacLearner(100, 64, 2, 1.0, batch_size=N, replay_capacity=1 << 20, lockstep_envs=N, seed=7)
            L.init_params(0)
            run = lambda: engine.sac_eval_run(ev, L, a.episodes)  # noqa: E731
        run()                                                                   # warm-up (first launches, allocations)
        res, dt = timed(run)
        steps = int(res["records"]["steps"].sum())
        r = {"episodes_per_s": res["n_records"] / dt, "env_steps_per_s": steps / dt, "us_per_iteration": 1e6 * dt / res["iterations"],
             "iterations": res["iterations"], "unfinished": res["unfinished"], "success": int((res["records"]["outcome"] == 1).sum())}
        tr = env_with_pool(True)
        tr.reset(0)
        if kind == "dqn":
            engine.train_run(tr, L, 4, 0.1, do_update=False, want_stats=False)
            ms = engine.train_profile(tr, L, a.train_iters, 0.1) if L.replay_size() > N else None
            engine.train_run(tr, L, 1, 0.1, do_update=False, want_stats=False)
            _, dtt = timed(lambda: engine.train_run(tr, L, a.train_iters, 0.1, do_update=False, want_stats=False))
            r["train_collect_us_per_iteration"] = 1e6 * dtt / a.train_iters
            if ms is not None:
                r["train_profile_act_us"] = 1e3 * float(ms[0]) / a.train_iters
                r["train_profile_env_step_us"] = 1e3 * float(ms[1]) / a.train_iters
        else:
            engine.sac_train_run(tr, L, 4, False, want_stats=False)
            _, dtt = timed(lambda: engine.sac_train_run(tr, L, a.train_iters, False, want_stats=False))
            r["train_collect_us_per_iteration"] = 1e6 * dtt / a.train_iters
        tr.close()
        out[kind] = r
        L.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
