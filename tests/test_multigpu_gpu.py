"""Two-rank NCCL data-parallel check (needs 2 GPUs; skipped otherwise): env/replay shards per rank,
gradient all-reduce between uavrl_learner_compute_grads and uavrl_learner_apply_grads keeps the replicas
bit-identical and equals a single learner fed the concatenated batch."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "oracle"))
import uavrl_b200
from uavrl_b200 import engine
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
g = np.load(os.path.join(%(root)r, "tests", "golden", "dqn_golden.npz"))
s = g["batch_s"].reshape(-1, 100); s2 = g["batch_s2"].reshape(-1, 100)
a = g["batch_a"].reshape(-1); r = g["batch_r"].reshape(-1); d = g["batch_d"].reshape(-1)
B = 128                                      # per-rank batch; rank r owns transitions [r*B, (r+1)*B)
def dev(x, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(x)).cuda(rank)
    return t if dt is None else t.to(dt)
sl = slice(rank * B, (rank + 1) * B)
idx = dev(np.arange(B, dtype=np.int32))
# data-parallel steps on explicit shards via compute_grads: enlarge the replay by one dummy transition
L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B, replay_capacity=B + 1, update_loop=2, device=rank)
L.set_params(g["ddqn_qvalue3_local0"], 0); L.set_params(g["ddqn_qvalue3_target0"], 1)
L.push(dev(s[sl]), dev(a[sl], torch.int32), dev(r[sl]), dev(s2[sl]), dev(d[sl], torch.uint8))
L.push(dev(s[:1]), dev(a[:1], torch.int32), dev(r[:1]), dev(s2[:1]), dev(d[:1], torch.uint8))
gt = L.grad_tensor()
for it in range(4):
    L.compute_grads(B * world, idx_tape=idx)
    dist.all_reduce(gt, op=dist.ReduceOp.SUM)
    L.apply_grads()
torch.cuda.synchronize()
p = torch.from_numpy(L.get_params(0)).cuda(rank); tgt = torch.from_numpy(L.get_params(1)).cuda(rank)
ps = [torch.zeros_like(p) for _ in range(world)]; dist.all_gather(ps, p)
if rank == 0:
    assert all(torch.equal(ps[0], q) for q in ps), "replicas diverged"
    # single learner on the concatenated batch
    S = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B * world, replay_capacity=1000, update_loop=2, device=0)
    S.set_params(g["ddqn_qvalue3_local0"], 0); S.set_params(g["ddqn_qvalue3_target0"], 1)
    n = B * world
    for it in range(4):
        S.update_batch(dev(s[:n]), dev(a[:n], torch.int32), dev(r[:n]), dev(s2[:n]), dev(d[:n]))
    torch.cuda.synchronize()
    np.testing.assert_allclose(L.get_params(0), S.get_params(0), atol=3e-6)
    np.testing.assert_allclose(L.get_params(1), S.get_params(1), atol=3e-6)
    assert L.counters() == S.counters() == (4, 4)
    print("DP_OK")
# ---- fused one-shot NVLink all-reduce + Adam (no NCCL on the update path) vs the NCCL path above
F = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=B, replay_capacity=B + 1, update_loop=2, device=rank)
F.set_params(g["ddqn_qvalue3_local0"], 0); F.set_params(g["ddqn_qvalue3_target0"], 1)
F.push(dev(s[sl]), dev(a[sl], torch.int32), dev(r[sl]), dev(s2[sl]), dev(d[sl], torch.uint8))
F.push(dev(s[:1]), dev(a[:1], torch.int32), dev(r[:1]), dev(s2[:1]), dev(d[:1], torch.uint8))
F.connect_peers(dist, rank, world)
loss = torch.zeros(1, device="cuda:%%d" %% rank)
for it in range(4):
    F.update_dp(B * world, idx_tape=idx, loss=loss)
torch.cuda.synchronize()
assert np.array_equal(F.get_params(0), L.get_params(0)), "fused all-reduce+Adam differs from NCCL all-reduce + Adam"
assert np.array_equal(F.get_params(1), L.get_params(1))
assert F.counters() == L.counters()
ls = [torch.zeros_like(loss) for _ in range(world)]; dist.all_gather(ls, loss)
assert all(torch.equal(ls[0], q) for q in ls) and float(loss) > 0          # every rank holds the same GLOBAL loss
if rank == 0:
    print("FUSED_OK")
dist.barrier(device_ids=[rank])
dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_data_parallel(tmp_path):
    script = tmp_path / "dp_worker.py"
    script.write_text(WORKER % {"root": ROOT})
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29577", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "DP_OK" in r.stdout and "FUSED_OK" in r.stdout


def test_fused_allreduce_pair_world1_equals_plain_update(dqn_golden):
    """The data-parallel optimiser kernel on ONE GPU (world = 1): reduce + push {tag : value} words into the local receive
    buffer, then poll for the current tag + rank-ordered sum + Adam -- must equal the single-GPU update (same partials, same
    Adam arithmetic), through hard updates and both parities of the double-buffered receive buffer; the loss is the batch
    loss."""
    import numpy as np
    from gpu_util import dev
    from uavrl_b200 import engine
    g = dqn_golden
    s = g["batch_s"].reshape(-1, 100)[:300]; s2 = g["batch_s2"].reshape(-1, 100)[:300]
    a = g["batch_a"].reshape(-1)[:300]; r = g["batch_r"].reshape(-1)[:300]; d = g["batch_d"].reshape(-1)[:300]
    Ls = []
    for _ in range(2):
        L = engine.Learner(100, [64, 64], 27, False, engine.ALGO_DDQN, batch_size=256, replay_capacity=300, update_loop=2)
        L.set_params(g["ddqn_qvalue3_local0"], 0); L.set_params(g["ddqn_qvalue3_target0"], 1)
        L.push(dev(s), dev(a, torch.int32), dev(r), dev(s2), dev(d, torch.uint8))
        Ls.append(L)
    Ls[1].connect_self()
    rng = np.random.default_rng(4)
    l0, l1 = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    for it in range(5):
        idx = dev(rng.permutation(300)[:256].astype(np.int32))
        Ls[0].update(idx_tape=idx, loss=l0)
        Ls[1].update_dp(256, idx_tape=idx, loss=l1)
        torch.cuda.synchronize()
        assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0))
        np.testing.assert_allclose(Ls[1].get_params(4), Ls[0].get_params(4), rtol=0, atol=1e-9)       # the reduced gradient
        np.testing.assert_allclose(Ls[1].get_params(0), Ls[0].get_params(0), rtol=0, atol=1e-7)
        np.testing.assert_allclose(Ls[1].get_params(1), Ls[0].get_params(1), rtol=0, atol=1e-7)
    assert Ls[0].counters() == Ls[1].counters() == (5, 5)
    for L in Ls:
        L.close()
