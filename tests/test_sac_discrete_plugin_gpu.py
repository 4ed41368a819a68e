"""The discrete SAC Trainer XML (configs/Trainer_SAC_discrete_B200.xml: IS_Continuous = 0, PolicyNet_SAC / QValueNet_SAC)
through the plug-ins: the trainer API, checkpoints in the reference's format, run_eposide on the 27-action step, the
actor aggregation, run_evaluation, and the pairings the env plug-in refuses."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from gpu_util import assert_same, env_dict, env_plugin

pytestmark = pytest.mark.gpu


def trainer_dict(tmp_path, **kw):
    from uavrl_b200.plugins import xmlconfig
    t = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", "Trainer_SAC_discrete_B200.xml"))["Trainer"]
    t.update(name="UAV_0", model_path=str(tmp_path), Batch_Size="64", replay_size="4096")
    t.update(kw)
    return t


def test_trainer_api_and_checkpoints(tmp_path):
    import importlib
    mod = importlib.import_module("uavrl_b200.plugins.SAC_Trainer_B200")
    g = np.load(os.path.join(GOLDEN, "sac_discrete_golden.npz"))
    tr = mod.SAC_Trainer_B200(trainer_dict(tmp_path))
    assert tr.IS_Continuous == 0 and tr._learner.discrete
    a = tr.get_action(g["sacd_s"][0][0], 0.1)
    assert isinstance(a, int) and 0 <= a < 27
    ab = tr.get_action(g["sacd_s"][0])
    assert ab.shape == (64,) and ab.dtype == np.int32 and ab.min() >= 0 and ab.max() < 27
    td = {"states": g["sacd_s"][0].tolist(), "actions": g["sacd_a"][0].tolist(), "next_states": g["sacd_s2"][0].tolist(),
          "rewards": g["sacd_r"][0].tolist(), "dones": g["sacd_d"][0].tolist()}
    res = tr.update(td)
    assert res["sum_epoch"] == 1 and np.isfinite(float(res["loss"][0]))
    assert tr.update({"states": [[]], "actions": [], "next_states": [], "rewards": [], "dones": []})["sum_epoch"] == 2
    tr.save()
    assert sorted(os.listdir(tmp_path)) == ["actor_SAC_UAV_0.pth", "critic_1_SAC_UAV_0.pth", "critic_2_SAC_UAV_0.pth"]
    keys = [str(k) for k in g["sacd_keys"]]
    shapes = [tuple(int(x) for x in s if x) for s in g["sacd_shapes"]]
    for i, f in enumerate(("actor", "critic_1")):
        ck = torch.load(os.path.join(tmp_path, "%s_SAC_UAV_0.pth" % f), weights_only=False)
        assert list(ck["model"]) == keys[6 * i:6 * i + 6]
        assert [tuple(v.shape) for v in ck["model"].values()] == shapes[6 * i:6 * i + 6]
        assert ck["epoch"] == 2 and set(ck["optimizer"]) == {"state", "param_groups"}
    tr2 = mod.SAC_Trainer_B200(trainer_dict(tmp_path))                   # Load_Mod in the constructor resumes, bit for bit
    for role in range(3):
        assert np.array_equal(tr2._learner.get_params(role), tr._learner.get_params(role))
        assert np.array_equal(tr2._learner.get_params(5 + role), tr._learner.get_params(5 + role))
        assert np.array_equal(tr2._learner.get_params(8 + role), tr._learner.get_params(8 + role))
    for role in (1, 2):
        assert np.array_equal(tr2._learner.get_params(role + 2), tr._learner.get_params(role))
    assert tr2.epoch == 2
    with pytest.raises(ValueError, match="prioritised replay is not available with IS_Continuous = 0"):
        mod.SAC_Trainer_B200(trainer_dict(tmp_path, IsPriority_Replay="1", lockstep_envs="64"))
    bad = trainer_dict(tmp_path)
    bad["actor"] = dict(bad["actor"], NetWork="PolicyNetContinuous_SAC")
    with pytest.raises(ValueError, match="IS_Continuous = 0 needs PolicyNet_SAC / QValueNet_SAC"):
        mod.SAC_Trainer_B200(bad)


@pytest.mark.parametrize("fl", [0, 1])
def test_run_eposide_federation_and_evaluation(tmp_path, fl):
    """Two run_eposide calls on the 27-action step (with Is_FL = Is_AC = 1: Federated_Learning_AC every episode), then
    run_evaluation with eval_mean_action 0 and 1, which change neither the trainer nor the training env."""
    extra = dict(Is_AC="1", Is_FL="1", FL_Loop="1") if fl else {}
    ed = env_dict("Trainer_SAC_discrete_B200.xml", "UAV_B200.xml", eval_episodes="24", eval_envs="8", **extra)
    with env_plugin(tmp_path / "Mod") as mod:
        cwd = os.getcwd()
        os.chdir(tmp_path)
        try:
            env = mod.PathPlan_City_B200(ed)
            L = env.Trainer._learner
            assert L.discrete and L.G == 8
            for _ in range(2):
                info = env.run_eposide(0.1)
                assert info["episodes"] >= 8 and np.isfinite(info["loss"])
            if fl:
                actors = L.get_params(0)
                assert all(np.array_equal(actors[0], actors[g]) for g in range(8))
            snap = lambda: [L.get_params(r) for r in range(11)] + [L.alpha()]  # noqa: E731
            before, state = snap(), env.batch.get_state()
            outs = []
            for mean in (0, 1):
                env.eval_mean_action = mean
                outs.append(env.run_evaluation())
        finally:
            os.chdir(cwd)
    for a, b in zip(before, snap()):
        assert_same(a, b, "trainer after run_evaluation")
    after = env.batch.get_state()
    for k in state:
        assert_same(after[k], state[k], "training env after run_evaluation: " + k)
    for out in outs:
        assert out["episodes"] + out["unfinished"] == 24 and out["success"] + out["lose"] == out["episodes"]


def test_env_refuses_mismatched_steps(tmp_path):
    """continuous SAC <-> the continuous step; discrete SAC and the DQN family <-> the 27-action step"""
    for trainer, agent in (("Trainer_SAC_discrete_B200.xml", "UAV_continuous_B200.xml"), ("Trainer_SAC_B200.xml", "UAV_B200.xml")):
        with env_plugin(tmp_path / "Mod") as mod:
            env = mod.PathPlan_City_B200(env_dict(trainer, agent))
            with pytest.raises(ValueError, match="continuous SAC needs update_function_name = update_PathPlan"):
                env.run_eposide(0.1)
