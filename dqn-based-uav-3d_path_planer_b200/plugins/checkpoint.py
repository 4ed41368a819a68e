"""The reference's .pth checkpoint of one network: torch.save of {'model': state_dict, 'optimizer': torch.optim.Adam
state_dict, 'epoch': int} (DuelingDQN_Trainer.py:41-84, SAC_Trainer.py:70-119).  A layout is the network's list of
(state_dict key, shape) in flat-parameter order (engine.Learner.layout, engine.SacLearner.layout)."""
import collections

import numpy as np
import torch


def flat(tensors):
    """Tensors or arrays concatenated into one flat float32 vector."""
    return np.concatenate([np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v, np.float32).ravel()
                           for v in tensors])


def _tensors(layout, x):
    """The layout's tensors of flat vector x, as CPU tensors that own their memory."""
    off = 0
    for _, shape in layout:
        k = int(np.prod(shape))
        yield torch.from_numpy(x[off:off + k].reshape(shape).copy())
        off += k


def model_dict(layout, x):
    """The network's state_dict holding flat parameters x."""
    return collections.OrderedDict(zip((key for key, _ in layout), _tensors(layout, x)))


def adam_dict(layout, m, v, step, lr):
    """torch.optim.Adam(params, lr).state_dict() after `step` steps with flat moments m (exp_avg) and v (exp_avg_sq)."""
    state = {i: {'step': torch.tensor(float(step)), 'exp_avg': a, 'exp_avg_sq': b}
             for i, (a, b) in enumerate(zip(_tensors(layout, m), _tensors(layout, v)))}
    return {'state': state, 'param_groups': [{'lr': lr, 'betas': (0.9, 0.999), 'eps': 1e-08, 'weight_decay': 0,
                                              'amsgrad': False, 'params': list(range(len(layout)))}]}


def adam_moments(layout, osd):
    """(exp_avg, exp_avg_sq, step) of an Adam state_dict of the network, flat; None when it holds no state.  Raises
    ValueError when the moments do not have the network's size."""
    st = osd.get('state', {})
    if not st:
        return None
    keys = sorted(st.keys())
    m, v = flat(st[k]['exp_avg'] for k in keys), flat(st[k]['exp_avg_sq'] for k in keys)
    n = sum(int(np.prod(shape)) for _, shape in layout)
    if m.size != n or v.size != n:
        raise ValueError("optimizer state holds %d / %d moments, the network has %d parameters" % (m.size, v.size, n))
    return m, v, int(float(st[keys[0]]['step']))


def read(path, layout):
    """(flat parameters, exp_avg or None, exp_avg_sq or None, Adam step or None, epoch) of a checkpoint file.  Raises
    ValueError when the file is not one of this network: its keys or a tensor's shape differ from the layout, as torch's
    strict load_state_dict refuses, or its optimizer state does not match the model."""
    ck = torch.load(path, weights_only=False, map_location='cpu')
    model = ck['model']
    if set(model) != {key for key, _ in layout}:
        raise ValueError("%s holds %s, the network has %s" % (path, list(model), [key for key, _ in layout]))
    for key, shape in layout:
        if tuple(model[key].shape) != shape:
            raise ValueError("%s: %s is %s, the network's is %s" % (path, key, tuple(model[key].shape), shape))
    m, v, step = adam_moments(layout, ck['optimizer']) or (None, None, None)
    return flat(model[key] for key, _ in layout), m, v, step, int(ck['epoch'])
