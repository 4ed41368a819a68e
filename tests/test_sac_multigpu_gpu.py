"""Two-rank data-parallel SAC (needs 2 GPUs; skipped otherwise): each rank fills its own ring from its own env shard with its
own seed; the split form with NCCL all-reduces between the phases and the fused update_replay_dp (connect_peers) give the
same bits, every replica is identical, and both match one learner fed the two ranks' batches concatenated."""
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import uavrl_b200
from uavrl_b200 import engine
import replay_restatement as R
from sac_restatement import HP
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
g = np.load(os.path.join(%(root)r, "tests", "golden", "env_golden.npz"))
dims, b, p = g["dims"], g["buildings"], g["uav_params"]
city = engine.City(dims[0], dims[1], dims[2], b)
params = engine.UavParams(p[0], p[1], p[2], 1.0, 12)
N, B, cap, seed = 64, 64, 4, 11 + rank
def pair():
    env = engine.EnvBatch(city, params, N, max_subgoals=64, device=rank, auto_reset=True)
    sc = env.make_scenarios(256, seed=20 + rank)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"]); env.reset(0)
    S = engine.SacLearner(batch_size=B, replay_capacity=N * cap, lockstep_envs=N, seed=seed, device=rank, **HP)
    S.init_params(4)                                          # same parameters on every rank
    engine.sac_train_run(env, S, 6, do_update=False)
    return env, S
(en, Sn), (ef, Sf) = pair(), pair()
Sf.connect_peers(dist, rank, world)
start = [Sn.get_params(r) for r in range(11)]
ln, lf = torch.zeros(4, device="cuda"), torch.zeros(4, device="cuda")
xs = (Sn.exchange_tensor(0), Sn.exchange_tensor(1))
STEPS = 3
for it in range(STEPS):
    Sn.critic_grads(B * world)
    dist.all_reduce(xs[0], op=dist.ReduceOp.SUM)
    Sn.apply_critic_grads()
    Sn.actor_grads()
    dist.all_reduce(xs[1], op=dist.ReduceOp.SUM)
    Sn.apply_actor_grads(ln)
    Sf.update_replay_dp(B * world, losses=lf)
torch.cuda.synchronize()
for r in range(14):
    a, f = Sn.get_params(r), Sf.get_params(r)
    assert (np.array_equal(a, f) if r >= 11 else np.array_equal(a.view(np.uint32), f.view(np.uint32))), ("nccl vs fused", r)
    t = torch.from_numpy(a).cuda(rank); ts = [torch.zeros_like(t) for _ in range(world)]; dist.all_gather(ts, t)
    assert all(torch.equal(ts[0], q) for q in ts), ("replicas diverged", r)
assert np.array_equal(Sn.alpha(), Sf.alpha()) and Sn.scalars() == Sf.scalars()
assert torch.equal(ln, lf)
print("SPLIT_FUSED_OK")
# one learner on the concatenated batches: every rank's rows of each epoch (restated sampler) and its Philox noise
ring = R.Ring(N * cap, N)
for _ in range(6):
    ring.commit()
E = Sn.scalars()["epoch"]
rows = []
for ep in range(E - STEPS + 1, E + 1):
    s, a, r_, s2, d = Sn.gather(R.sample(seed, ep, ring.count, B))
    c1, c2 = R.sac_update_ctrs(ep)
    flat = np.concatenate([s.ravel(), a.ravel(), r_, s2.ravel(), d.astype(np.float32), R.sac_noise(seed, c1, B).ravel().astype(np.float32),
                           R.sac_noise(seed, c2, B).ravel().astype(np.float32)])
    t = torch.from_numpy(flat).cuda(rank); ts = [torch.zeros_like(t) for _ in range(world)]; dist.all_gather(ts, t)
    rows.append([q.cpu().numpy() for q in ts])
if rank == 0:
    X = engine.SacLearner(batch_size=B * world, seed=1, device=0, **HP)
    for r in range(11):
        X.set_params(r, start[r])
    o = 100
    cuts = np.cumsum([B * o, B * 2, B, B * o, B, B * 2, B * 2])
    for per_rank in rows:
        parts = [np.split(q, cuts[:-1]) for q in per_rank]
        cat = lambda k, shape: torch.from_numpy(np.concatenate([pp[k] for pp in parts]).reshape(shape)).cuda(0)
        n = B * world
        X.update_batch(cat(0, (n, o)), cat(1, (n, 2)), cat(2, (n,)), cat(3, (n, o)), cat(4, (n,)), cat(5, (n, 2)), cat(6, (n, 2)))
    torch.cuda.synchronize()
    for r, lr in ((0, HP["actor_lr"]), (1, HP["critic_lr"]), (2, HP["critic_lr"])):
        # the kernels' Philox noise and the float64 restatement's differ by a few ulp: each Adam step moves a parameter by at
        # most about lr, so replicas and the single learner agree to well inside 2 lr per step
        np.testing.assert_allclose(Sn.get_params(r), X.get_params(r), rtol=0, atol=2 * lr * STEPS)
    assert Sn.scalars()["adam_step"] == X.scalars()["adam_step"] == STEPS
    print("SINGLE_OK")
dist.barrier(device_ids=[rank])
dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_sac_data_parallel(tmp_path):
    script = tmp_path / "sac_dp_worker.py"
    script.write_text(WORKER % {"root": ROOT})
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29579", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SPLIT_FUSED_OK" in r.stdout and "SINGLE_OK" in r.stdout
