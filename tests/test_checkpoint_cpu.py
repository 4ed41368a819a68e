"""Parameter layouts and the reference's .pth checkpoint format, without a GPU: every network's layout names and shapes its
tensors as the reference's classes do (BaseClass/BaseCNN.py) and adds up to the parameter count of the C side's
build_mlp; a checkpoint round-trips bit for bit; a file of another network is refused."""
import types

import numpy as np
import pytest
import torch

import uavrl_b200  # noqa: F401
from uavrl_b200 import engine
from uavrl_b200.plugins import checkpoint

# weight shapes of the reference's classes at w = 100, hiden_dim = 64, output = 27 (action_dim = 2 for SAC); every
# weight has a bias of its first dimension
Q_WEIGHTS = {
    "Qnet2": [("fc1", (64, 100)), ("fc2", (27, 64))],
    "QValueNet_SAC": [("fc1", (64, 100)), ("fc2", (64, 64)), ("fc3", (27, 64))],
    "VAnet2": [("fc1", (64, 100)), ("fc_A", (27, 64)), ("fc_V", (1, 64))],
    "VAnet3": [("fc1", (128, 100)), ("fc2", (64, 128)), ("fc_A", (27, 64)), ("fc_V", (1, 64))],
    "VAnet4": [("fc1", (128, 100)), ("fc2", (64, 128)), ("fc3", (64, 64)), ("fc_A", (27, 64)), ("fc_V", (1, 64))],
    "VAnet5": [("fc1", (128, 100)), ("fc2", (64, 128)), ("fc3", (64, 64)), ("fc4", (64, 64)), ("fc_A", (27, 64)),
               ("fc_V", (1, 64))],
}
SAC_WEIGHTS = {
    0: [("fc1", (64, 100)), ("fc_mu", (2, 64)), ("fc_std", (2, 64))],                # PolicyNetContinuous_SAC
    1: [("fc1", (64, 102)), ("fc2", (64, 64)), ("fc_out", (2, 64))],                 # QValueNetContinuous_SAC
}


def expand(weights):
    return [(k, s) for nm, w in weights for k, s in ((nm + ".weight", w), (nm + ".bias", (w[0],)))]


def build_mlp_count(in_dim, hidden, head_main, head_extra):
    """Parameter count of csrc/net.cuh build_mlp: every trunk layer, then the head with its extra rows."""
    P, fan_in = 0, in_dim
    for h in hidden:
        P, fan_in = P + h * fan_in + h, h
    return P + (head_main + head_extra) * (fan_in + 1)


def q_learner(kind, h=64, in_dim=100, n_actions=27):
    hidden_fn, dueling = engine.NET_KINDS[kind]
    L = engine.Learner.__new__(engine.Learner)           # the layout needs no device
    L.in_dim, L.hidden, L.n_actions, L.dueling = in_dim, hidden_fn(h), n_actions, bool(dueling)
    return L


def sac_learner(obs_dim=100, hidden=64, act_dim=2):
    S = engine.SacLearner.__new__(engine.SacLearner)
    S.cfg = types.SimpleNamespace(obs_dim=obs_dim, hidden=hidden, act_dim=act_dim)
    return S


def size(layout):
    return sum(int(np.prod(s)) for _, s in layout)


@pytest.mark.parametrize("kind", sorted(engine.NET_KINDS))
def test_q_layout_is_the_reference_network(kind):
    assert sorted(Q_WEIGHTS) == sorted(engine.NET_KINDS)
    L = q_learner(kind)
    assert L.layout() == expand(Q_WEIGHTS[kind])
    assert size(L.layout()) == build_mlp_count(100, L.hidden, 27, int(L.dueling))
    for h in (1, 24, 128):                             # other widths: the C side's count still holds
        L = q_learner(kind, h, 37, 5)
        assert size(L.layout()) == build_mlp_count(37, L.hidden, 5, int(L.dueling))


def test_shipped_q_network_count():
    assert size(q_learner("QValueNet_SAC").layout()) == 12379           # 100-64-64-27 (DESIGN section 4)


def test_sac_layout_is_the_reference_network():
    S = sac_learner()
    assert S.layout(0) == expand(SAC_WEIGHTS[0])
    for role in (1, 2, 3, 4):
        assert S.layout(role) == expand(SAC_WEIGHTS[1])
    assert size(S.layout(0)) == build_mlp_count(100, [64], 2, 2) == 6724           # fc1 -> {fc_mu ; fc_std}
    assert size(S.layout(1)) == build_mlp_count(102, [64, 64], 2, 0) == 10882      # fc1 -> fc2 -> fc_out


def test_init_draw_is_linear_default_init():
    """U(+-1/sqrt(fan_in)) per tensor, with the bias of a layer bounded by its weight's fan-in, drawn in layout order."""
    lay = q_learner("VAnet3").layout()
    g = torch.Generator().manual_seed(3)
    flat = engine.init_draw(lay, g)
    assert flat.dtype == np.float32 and flat.size == size(lay)
    off, fan_in = 0, None
    for key, shape in lay:
        n = int(np.prod(shape))
        fan_in = shape[1] if key.endswith(".weight") else fan_in
        part = np.abs(flat[off:off + n])
        assert part.max() <= 1 / np.sqrt(fan_in), key
        assert n < 1000 or part.max() > 0.99 / np.sqrt(fan_in), key     # the bound, not a smaller one
        off += n
    again = engine.init_draw(lay, torch.Generator().manual_seed(3))
    assert again.tobytes() == flat.tobytes()


def save_file(path, layout, rng, epoch=17, step=9, lr=5e-4):
    n = size(layout)
    x, m, v = (rng.normal(0, 1, n).astype(np.float32) for _ in range(3))
    torch.save({'model': checkpoint.model_dict(layout, x), 'optimizer': checkpoint.adam_dict(layout, m, v, step, lr),
                'epoch': epoch}, path)
    return x, m, v


@pytest.mark.parametrize("net", ["VAnet3", "Qnet2", "sac_actor", "sac_critic"])
def test_round_trip_bit_for_bit(tmp_path, net):
    lay = {"sac_actor": sac_learner().layout(0), "sac_critic": sac_learner().layout(1)}.get(net) or q_learner(net).layout()
    path = str(tmp_path / "ck.pth")
    x, m, v = save_file(path, lay, np.random.default_rng(1))
    ck = torch.load(path, weights_only=False)
    assert list(ck["model"]) == [k for k, _ in lay]
    assert [tuple(t.shape) for t in ck["model"].values()] == [s for _, s in lay]
    group = ck["optimizer"]["param_groups"][0]
    assert group == {'lr': 5e-4, 'betas': (0.9, 0.999), 'eps': 1e-08, 'weight_decay': 0, 'amsgrad': False,
                     'params': list(range(len(lay)))}
    got = checkpoint.read(path, lay)
    for a, b in zip(got[:3], (x, m, v)):
        assert a.dtype == np.float32 and a.tobytes() == b.tobytes()
    assert got[3:] == (9, 17)


def test_round_trip_into_a_torch_module(tmp_path):
    """A state_dict of the layout loads strictly into the reference's module shape, and its Adam state into torch's Adam."""
    lay = q_learner("VAnet2").layout()
    x, m, v = save_file(str(tmp_path / "ck.pth"), lay, np.random.default_rng(2))
    net = torch.nn.ModuleDict({"fc1": torch.nn.Linear(100, 64), "fc_A": torch.nn.Linear(64, 27), "fc_V": torch.nn.Linear(64, 1)})
    ck = torch.load(str(tmp_path / "ck.pth"), weights_only=False)
    net.load_state_dict(ck["model"])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck["optimizer"])
    assert checkpoint.flat(net.parameters()).tobytes() == x.tobytes()
    assert checkpoint.adam_moments(lay, opt.state_dict())[0].tobytes() == m.tobytes()


def test_optimizer_without_state(tmp_path):
    lay = q_learner("Qnet2").layout()
    path = str(tmp_path / "ck.pth")
    x = np.arange(size(lay), dtype=np.float32)
    torch.save({'model': checkpoint.model_dict(lay, x), 'optimizer': {'state': {}, 'param_groups': []}, 'epoch': 3}, path)
    flat, m, v, step, epoch = checkpoint.read(path, lay)
    assert flat.tobytes() == x.tobytes() and (m, v, step, epoch) == (None, None, None, 3)


def test_read_refuses_another_network(tmp_path):
    lay = q_learner("VAnet3").layout()
    rng = np.random.default_rng(3)
    path = str(tmp_path / "ck.pth")
    x, m, v = save_file(path, lay, rng)
    good = torch.load(path, weights_only=False)
    small = q_learner("VAnet3", h=32).layout()
    n = size(small)

    def refused(match, model=good["model"], osd=good["optimizer"]):
        torch.save({'model': model, 'optimizer': osd, 'epoch': 1}, path)
        with pytest.raises(ValueError, match=match):
            checkpoint.read(path, lay)

    refused("fc_Adv.weight", {("fc_Adv" + k[4:] if k.startswith("fc_A.") else k): t for k, t in good["model"].items()})
    refused(r"fc1.weight is \(100, 128\)", dict(good["model"], **{"fc1.weight": good["model"]["fc1.weight"].t().contiguous()}))
    refused("fc1.weight", checkpoint.model_dict(small, x[:n]))                     # a smaller network of the same kind
    refused("optimizer state", osd=checkpoint.adam_dict(small, m[:n], v[:n], 1, 1e-3))
    torch.save(good, path)
    assert checkpoint.read(path, lay)[0].tobytes() == x.tobytes()
