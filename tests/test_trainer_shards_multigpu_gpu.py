"""The env plug-in with <shard_over_ranks>1</shard_over_ranks> on W >= 2 GPUs (torchrun; skipped with fewer GPUs):
num_trainers = num_UAV = 8 and Is_FL = 1, FL_Loop = 1, two episodes each for a DQN-family XML and a SAC Is_AC = 1 XML.
Every rank's trainers equal the matching trainers of the one-GPU plug-in run, the integer counts of the result dicts are
equal, score and loss agree to float rounding, and the checkpoint directories of the two runs load into each other."""
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
from gpu_util import env_dict, env_plugin
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
out = %(out)r
INTS = ("success", "lose", "normal", "sum_epoch", "step", "env_steps", "updates", "collisions", "episodes")

def rows(tr, sac):
    L = tr._learner
    return [L.get_params(w).reshape(L.G, -1) for w in (range(11) if sac else range(4))]

def gathered(mine):
    allr = []
    for a in mine:
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda(rank)
        ts = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(ts, t)
        allr.append(torch.cat(ts).cpu().numpy())
    return allr

for xml, agent, ac in (("Trainer_DDQN_B200.xml", None, "0"), ("Trainer_SAC_B200.xml", "UAV_continuous_B200.xml", "1")):
    sac = ac == "1"
    kw = dict(Is_FL="1", FL_Loop="1", Is_AC=ac)
    with env_plugin(os.path.join(out, "unused")) as mod:
        env = mod.PathPlan_City_B200(env_dict(xml, agent, shard_over_ranks="1", **kw))
        assert env.n_local == 8 // world and env.Trainer._learner.G == 8 // world
        res = [dict(env.run_eposide(0.3)) for _ in range(2)]
        mine = rows(env.Trainer, sac)
        dshard = os.path.join(out, "shard_" + xml)
        env.Trainer.save(dshard)
        allr = gathered(mine)
        dist.barrier(device_ids=[rank])
        if rank == 0:
            one = mod.PathPlan_City_B200(env_dict(xml, agent, **kw))
            ref = [dict(one.run_eposide(0.3)) for _ in range(2)]
            for a, b in zip(allr, rows(one.Trainer, sac)):
                assert np.array_equal(a, b), xml
            for r1, r2 in zip(res, ref):
                for k in INTS:
                    assert r1[k] == r2[k], (xml, k, r1[k], r2[k])
                np.testing.assert_allclose(r1["score"], r2["score"], rtol=1e-9)
                np.testing.assert_allclose(r1["loss"], r2["loss"], rtol=1e-5, atol=1e-7)
            # checkpoints: the shards' directory loads into a one-GPU trainer, and the one-GPU directory into the shards' layout
            fresh = mod.PathPlan_City_B200(env_dict(xml, agent, **kw))
            fresh.Trainer.model_dir = dshard
            fresh.Trainer.Load_Mod(dshard) if not sac else fresh.Trainer.Load_Mod()
            for a, b in zip(rows(fresh.Trainer, sac)[:3], rows(one.Trainer, sac)[:3]):
                assert np.array_equal(a, b), ("load shards", xml)
            one.Trainer.save(os.path.join(out, "one_" + xml))
        dist.barrier(device_ids=[rank])
        back = mod.PathPlan_City_B200(env_dict(xml, agent, shard_over_ranks="1", **kw))
        back.Trainer.model_dir = os.path.join(out, "one_" + xml)
        back.Trainer.Load_Mod(back.Trainer.model_dir) if not sac else back.Trainer.Load_Mod()
        for a, b in zip(rows(back.Trainer, sac)[:3], mine[:3]):
            assert np.array_equal(a, b), ("load one-GPU", xml)
    print("SHARDED_OK", xml)
dist.barrier(device_ids=[rank])
dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_env_plugin_sharded_over_ranks(tmp_path):
    script = tmp_path / "shard_worker.py"
    script.write_text(WORKER % {"root": ROOT, "out": str(tmp_path)})
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29581", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("SHARDED_OK") == 4
