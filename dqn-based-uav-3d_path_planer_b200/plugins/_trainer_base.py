"""Shared implementation of the DQN-family trainer plug-ins (the reference's BaseTrainer + the three
concrete trainers): same constructor dict, attributes and methods; the math runs in libuavrl_b200."""
import os

import numpy as np
import torch

import uavrl_b200  # noqa: F401  (repository root must be on sys.path)
from uavrl_b200 import engine
from uavrl_b200.plugins import checkpoint
from uavrl_b200.plugins.xmlconfig import None2Value

# BaseClass/BaseCNN.py class name -> (hidden widths as a function of hiden_dim, dueling flag)
NETWORKS = engine.NET_KINDS


class _ReplayFacade:
    """ReplayMemory surface the env uses (BaseClass/replay_buffer.py:28-54): add(), len(buffer), sample2()."""

    def __init__(self, trainer):
        self._t = trainer
        self.capacity = trainer.replay_size
        self.memory = self          # len(trainer.replay_memory.memory) is what learn_off_policy gates on

    class _Len:
        def __init__(self, t):
            self._t = t

        def __len__(self):
            return self._t._learner.replay_size()

    @property
    def buffer(self):
        return _ReplayFacade._Len(self._t)

    def __len__(self):
        return self._t._learner.replay_size()

    def add(self, state, action, reward, next_state, done):
        self._t._add([state], [action], [reward], [next_state], [done])

    def add_batch(self, states, actions, rewards, next_states, dones):
        self._t._add(states, actions, rewards, next_states, dones)

    def sample2(self, batch_size):
        """random.sample(buffer, B) + stacking (replay_buffer.py:48-51); indices drawn on the host.  With
        IsPriority_Replay: ReplayTree.sample2 (:186-213) -- stratified draw on the device, returns the tree indices
        (slot + capacity - 1) and the importance weights as the 6th / 7th element."""
        if self._t.IsPriority_Replay:
            t = self._t
            slots, w = t._learner.per_sample(int(batch_size))
            slots = slots.cpu().numpy().astype(np.int64)
            n, cap = t._learner.replay_size(), t.replay_size
            oldest = (t._head - n) % cap
            s, a, r, s2, d = t._learner.gather((slots - oldest) % cap)
            return (s, tuple(a.tolist()), tuple(r.tolist()), s2, tuple(bool(x) for x in d), (slots + cap - 1).tolist(),
                    w.cpu().numpy().astype(np.float64))
        n = self._t._learner.replay_size()
        idx = self._t._rng.choice(n, int(batch_size), replace=False)       # random.sample: distinct, uniform
        s, a, r, s2, d = self._t._learner.gather(idx)
        return s, tuple(a.tolist()), tuple(r.tolist()), s2, tuple(bool(x) for x in d), None, None


class TrainerB200:
    ALGO = engine.ALGO_DQN
    TAG = ""                      # file-name tag of the reference's save(): q_local_<TAG><name>.pth

    def __init__(self, param: dict) -> None:
        # BaseTrainer.__init__ (BaseClass/BaseTrainer.py:20-47)
        self.h = int(None2Value(param.get('h'), 1))
        self.w = int(None2Value(param.get('w'), 1))
        self.channel = int(None2Value(param.get('channel'), 1))
        self.output = int(None2Value(param.get('output'), 1))
        self.name = param.get('name')
        self.replay_size = int(None2Value(param.get('replay_size'), 1000))
        self.LEARNING_RATE = float(None2Value(param.get('LEARNING_RATE'), 0.001))
        self.Batch_Size = int(None2Value(param.get('Batch_Size'), 128))
        self.gamma = float(None2Value(param.get('gamma'), 0.99))
        self.max_epoch = int(None2Value(param.get('max_epoch'), 100000))
        self.save_loop = int(None2Value(param.get('save_loop'), 10))
        self.Is_Train = int(None2Value(param.get("Is_Train"), 1))
        self.Update_loop = int(None2Value(param.get('Update_loop'), 3))
        self.act_num = self.output
        net = param.get('NetWork')
        if net not in NETWORKS:
            raise ValueError("NetWork %r is not an MLP Q-network of the hot path (%s)" % (net, sorted(NETWORKS)))
        hid = int(None2Value(param.get('hiden_dim'), 64))
        hidden_fn, dueling = NETWORKS[net]
        self.network = net
        self.device_index = int(None2Value(param.get('device'), 0))
        self.lockstep_envs = int(None2Value(param.get('lockstep_envs'), 0))
        # n_trainers = G > 1: one independent trainer per block of lockstep_envs / G UAVs (the reference's Trainer per UAV,
        # PathPlan_City.py:59-69), each with its own replay_size transitions; trainer g is named UAV_<g * lockstep_envs / G>
        self.n_trainers = int(None2Value(param.get('n_trainers'), 1))
        G = self.n_trainers
        self.names = [self.name] if G == 1 else ['UAV_%d' % (g * (self.lockstep_envs // G)) for g in range(G)]
        self._learner = engine.Learner(self.w, hidden_fn(hid), self.output, dueling, self.ALGO, lr=self.LEARNING_RATE,
                                       gamma=self.gamma, batch_size=self.Batch_Size, update_loop=self.Update_loop,
                                       replay_capacity=self.replay_size * G, lockstep_envs=self.lockstep_envs,
                                       seed=int(None2Value(param.get('seed'), 42)), device=self.device_index, trainers=G)
        self._learner.init_params(int(None2Value(param.get('seed'), 42)))
        self._dev = self._learner.device
        self._loss = torch.zeros(G, device=self._dev)
        self.loss = 0
        self._rng = np.random.default_rng([int(None2Value(param.get('seed'), 42)), sum(map(ord, str(self.name)))])
        self._learner.set_is_train(self.Is_Train)        # the lockstep loops read it (get_action greedy when 0)
        self._pin = {}                                   # pinned host staging, by (tag, slot)
        self._pin_turn = 0
        self._dist, self._rank, self._world = None, 0, 1
        self._head = 0                                   # next replay slot (SumTree.data_pointer)
        self.IsPriority_Replay = int(None2Value(param.get('IsPriority_Replay'), 0))
        if self.IsPriority_Replay:
            if self.lockstep_envs == 0 and self.replay_size > 4 * 1024 * 1024:
                raise ValueError("prioritised replay supports at most 4194304 slots")
            # ReplayTree constants (replay_buffer.py:141-148); several trainers: one tree per trainer, as each reference
            # Trainer owns its ReplayTree (BaseTrainer.py:39).  The host-driven paths below stay single-trainer.
            if G > 1:
                self._learner.per_enable_trainers()
            else:
                self._learner.per_enable()
        self.replay_memory = _ReplayFacade(self)
        self.model_dir = None2Value(param.get('model_path'), None)
        self.Load_Mod(self.model_dir)

    # ---- reference attribute: epoch counts update() calls (DuelingDQN_Trainer.py:152)
    @property
    def epoch(self):
        return self._learner.counters()[0]

    # ---- host <-> device staging.  Arrays this plug-in hands out (actions; the env plug-in's observations) are numpy views
    # of PINNED buffers taken round-robin from a ring of 4, so when the caller passes them back (state -> get_action ->
    # replay add, as PathPlan_City.run_thread_OffPolicy does) the upload is a direct DMA.  A returned array stays valid for
    # the next 3 calls that return the same kind of array.
    def _pinned(self, tag, shape, dtype):
        self._pin_turn = (self._pin_turn + 1) % 4
        key = (tag, self._pin_turn, tuple(shape), dtype)
        buf = self._pin.get(key)
        if buf is None:
            buf = self._pin[key] = torch.empty(tuple(shape), dtype=dtype, pin_memory=True)
        return buf

    def _h2d(self, arr):
        """numpy array (pinned or pageable) -> device tensor on the current stream, without a host synchronisation."""
        return torch.from_numpy(arr).to(self._dev, non_blocking=True)

    def attach_dist(self, dist, rank, world):
        """Data-parallel training, one process per GPU: learn_off_policy() then runs the fused one-shot NVLink all-reduce +
        Adam (uavrl_learner_update_dp) on this rank's replay shard; replicas stay bit-identical."""
        self._dist, self._rank, self._world = dist, int(rank), int(world)
        if self._world > 1:
            self._learner.connect_peers(dist, self._rank, self._world)

    # ---- acting
    def get_action(self, state, eps):
        """DuelingDQN_Trainer.get_action (:86-97).  state: [w] -> python int, or [N, w] -> int32 array."""
        s = np.ascontiguousarray(state, np.float32)
        single = s.ndim == 1
        s = s.reshape(-1, self.w)
        a = self._learner.act(self._h2d(s), float(eps), is_train=bool(self.Is_Train))
        out = self._pinned("act", (s.shape[0],), torch.int32)
        out.copy_(a, non_blocking=True)
        torch.cuda.current_stream(self._dev).synchronize()
        return int(out[0]) if single else out.numpy()

    def get_q(self, state):
        s = torch.from_numpy(np.ascontiguousarray(state, np.float32).reshape(-1, self.w)).to(self._dev)
        return self._learner.act(s, 0.0, want_q=True)[1].cpu().numpy()

    # ---- replay
    def _add(self, states, actions, rewards, next_states, dones):
        s = self._h2d(np.ascontiguousarray(states, np.float32).reshape(-1, self.w))
        s2 = self._h2d(np.ascontiguousarray(next_states, np.float32).reshape(-1, self.w))
        a = self._h2d(np.ascontiguousarray(actions, np.int32).reshape(-1))
        r = self._h2d(np.ascontiguousarray(rewards, np.float32).reshape(-1))
        d = self._h2d(np.ascontiguousarray(dones).astype(np.uint8, copy=False).reshape(-1))
        self._learner.push(s, a, r, s2, d)
        slots = (self._head + np.arange(s.shape[0])) % self.replay_size
        self._head = int((self._head + s.shape[0]) % self.replay_size)
        return slots

    def Push_Replay(self, Experience, error=None):
        """(state, action, reward, next_state, done) tuple, tensors or arrays (PathPlan_City.py:374-379)."""
        s, a, r, s2, d = [x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x) for x in Experience]
        slots = self._add(s, a, r, s2, d)
        if self.IsPriority_Replay and error is not None:           # ReplayTree.push(sample, error) (:152-154)
            e = error.detach().cpu().numpy() if isinstance(error, torch.Tensor) else np.asarray(error)
            e = np.abs(e.astype(np.float32)).reshape(-1)
            e = np.full(len(slots), e[0], np.float32) if e.size == 1 else e
            self._learner.per_set_errors(torch.from_numpy(slots.astype(np.int32)).to(self._dev),
                                         torch.from_numpy(np.ascontiguousarray(e)).to(self._dev), clip=False)

    # ---- learning
    def update(self, transition_dict):
        """Trainer.update(transition_dict) (DuelingDQN_Trainer.py:150-190): explicit batch."""
        states = transition_dict['states']
        if isinstance(states, list) and len(states) == 0:      # :155-156, epoch still counts (:152)
            e, t = self._learner.counters()
            self._learner.set_counters(e + 1, t)
            return {'sum_epoch': self.epoch, 'loss': self.loss}
        if self.Is_Train:
            dev = self._dev
            s = self._h2d(np.ascontiguousarray(states, np.float32))
            s2 = self._h2d(np.ascontiguousarray(transition_dict['next_states'], np.float32))
            a = self._h2d(np.asarray(transition_dict['actions'], np.float32).astype(np.int32).reshape(-1))
            r = self._h2d(np.ascontiguousarray(transition_dict['rewards'], np.float32).reshape(-1))
            d = self._h2d(np.ascontiguousarray(transition_dict['dones'], np.float32).reshape(-1))
            idx, wts = transition_dict.get('idx'), transition_dict.get('weights')
            if self.IsPriority_Replay and idx is not None and wts is not None:
                # importance weights in the loss, then ReplayTree.batch_update(tree_idx, |TD error|) (SAC_Trainer.py:336-352)
                w = torch.as_tensor(np.asarray(wts, np.float32).reshape(-1)).to(dev)
                ae = torch.zeros(s.shape[0], dtype=torch.float32, device=dev)
                self._learner.update_batch_per(s, a, r, s2, d, w, ae, self._loss)
                slots = torch.as_tensor((np.asarray(idx, np.int64).reshape(-1) - (self.replay_size - 1)).astype(np.int32)).to(dev)
                self._learner.per_set_errors(slots, ae, clip=True)
            else:
                self._learner.update_batch(s, a, r, s2, d, self._loss)
            self.loss = self._loss            # a 1-element tensor, like the reference's `self.loss = loss`
        else:                                 # self.epoch += 1 is unconditional (:152); the C update did it when training
            e, t = self._learner.counters()
            self._learner.set_counters(e + 1, t)
            if self.Update_loop > 0 and (e + 1) % self.Update_loop == 0:
                self._learner.hard_update()   # :183-184 runs whether or not Is_Train
        self._maybe_save()
        return {'sum_epoch': self.epoch, 'loss': self.loss}

    def learn_off_policy(self):
        """DQN_Trainer/DDQN_Trainer.learn_off_policy (:85-136 / :72-117): sample from the replay, update."""
        if self._learner.replay_size() > self.Batch_Size and self.Is_Train:
            if self._world > 1:
                self._learner.update_dp(self.Batch_Size * self._world, loss=self._loss)
            else:
                self._learner.update(loss=self._loss)
            self.loss = self._loss
        else:
            e, t = self._learner.counters()
            self._learner.set_counters(e + 1, t)
        self._maybe_save()
        return {'sum_epoch': self.epoch, 'loss': self.loss}

    def hard_update(self):
        self._learner.hard_update()

    def _learner_reset_lockstep(self):
        """An explicit env reset invalidates the lockstep ring's current observation frame."""
        if self.lockstep_envs > 0:
            self._learner.lockstep_restart()

    def replace_param(self, target):
        """Copy another trainer's / torch module's parameters into q_local (:204-207)."""
        self._learner.set_params(_flat_from(target), 0)

    def replace_target_param(self, target):
        self._learner.set_params(_flat_from(target), 1)

    # ---- checkpoints: the reference's {'model', 'optimizer', 'epoch'} .pth files (DuelingDQN_Trainer.py:41-84)
    def _rows(self, which):
        """Vector `which` of every trainer, (G, P), in ONE device read: checkpoints of many trainers slice these rows
        instead of reading the whole [G][P] vector once per trainer."""
        return self._learner.get_params(which).reshape(self.n_trainers, -1)

    def state_dict(self, which=0, g=0, flat=None):
        """Trainer g's network `which` (0 q_local, 1 q_target) as a state_dict; `flat` = its row when already on the host."""
        return checkpoint.model_dict(self._learner.layout(), self._rows(which)[g] if flat is None else flat)

    def load_state_dict(self, sd, which=0, g=0):
        flat = checkpoint.flat(sd.values())
        if self.n_trainers > 1:                 # trainer g's row of the [G][P] parameters
            rows = self._rows(which)
            rows[g] = flat
            flat = rows
        self._learner.set_params(flat, which)

    def optimizer_state_dict(self, g=0, m=None, v=None):
        """torch.optim.Adam state_dict of trainer g; m / v = its exp_avg / exp_avg_sq rows when already on the host."""
        m = self._rows(2)[g] if m is None else m
        v = self._rows(3)[g] if v is None else v
        return checkpoint.adam_dict(self._learner.layout(), m, v, self._learner.counters()[1], self.LEARNING_RATE)

    def load_optimizer_state_dict(self, osd, g=0):
        mvs = checkpoint.adam_moments(self._learner.layout(), osd)
        if mvs is None:
            return
        for which, x in ((2, mvs[0]), (3, mvs[1])):
            rows = self._rows(which)
            rows[g] = x
            self._learner.set_params(rows, which)
        self._learner.set_counters(self._learner.counters()[0], mvs[2])

    def _paths(self, directory, g=0):
        return (os.path.join(directory, 'q_target_%s%s.pth' % (self.TAG, self.names[g])),
                os.path.join(directory, 'q_local_%s%s.pth' % (self.TAG, self.names[g])))

    def save(self, directory=None):
        """One q_target / q_local file pair per trainer, named after the trainer (the reference's per-UAV files).  Each of the
        four vectors is read from the device once for all trainers."""
        directory = directory or self.model_dir or os.path.join(os.getcwd(), 'Mod')
        os.makedirs(directory, exist_ok=True)
        local, target, m, v = (self._rows(w) for w in range(4))
        epoch = self.epoch
        for g in range(self.n_trainers):
            pt, pl = self._paths(directory, g)
            osd = self.optimizer_state_dict(g, m[g], v[g])
            torch.save({'model': self.state_dict(1, g, target[g]), 'optimizer': osd, 'epoch': epoch}, pt)
            torch.save({'model': self.state_dict(0, g, local[g]), 'optimizer': osd, 'epoch': epoch}, pl)

    def Load_Mod(self, Mod_path=None):
        """DuelingDQN_Trainer.Load_Mod (:40-69): <root>/Mod by default; a given Mod_path is tried as written and, like the
        reference's `root + Mod_path`, relative to the working directory.  Every trainer whose file pair exists and parses
        as this network is restored into host copies of the four vectors, which go to the device once each; a trainer
        whose files do not parse is left as it is."""
        directory = Mod_path or os.path.join(os.getcwd(), 'Mod')
        if Mod_path and not os.path.isdir(directory) and os.path.isdir(os.path.join(os.getcwd(), Mod_path.lstrip('/'))):
            directory = os.path.join(os.getcwd(), Mod_path.lstrip('/'))
        rows, epoch, step = None, None, None
        for g in range(self.n_trainers):
            pt, pl = self._paths(directory, g)
            if not (os.path.exists(pt) and os.path.exists(pl)):
                continue
            try:
                tgt = checkpoint.read(pt, self._learner.layout())[0]
                loc, m, v, st, ep = checkpoint.read(pl, self._learner.layout())
            except Exception as e:          # the reference prints and carries on (:56-57); nothing was applied
                print(e.args)
                continue
            if rows is None:
                rows = [self._rows(w) for w in range(4)]
            rows[0][g], rows[1][g] = loc, tgt
            if m is not None:
                rows[2][g], rows[3][g], step = m, v, st
            epoch = ep
        if rows is None:
            return
        for w in range(4):
            self._learner.set_params(rows[w], w)
        e, t = self._learner.counters()
        self._learner.set_counters(epoch, t if step is None else step)

    def _maybe_save(self):
        if self.save_loop > 0 and self.epoch % self.save_loop == 0:
            self.save()

    # ---- setters of the reference surface
    def set_replay_size(self, replay_size: int):
        self.replay_size = replay_size

    def set_LEARNING_RATE(self, LEARNING_RATE: float):
        self.LEARNING_RATE = LEARNING_RATE

    def set_Batch_Size(self, Batch_Size: int):
        self.Batch_Size = Batch_Size

    def set_gamma(self, gamma: float):
        self.gamma = gamma

    def set_max_epoch(self, max_epoch: int):
        self.max_epoch = max_epoch

    def set_save_loop(self, save_loop: int):
        self.save_loop = save_loop


def _flat_from(obj):
    if isinstance(obj, TrainerB200):
        return obj._learner.get_params(0)
    if hasattr(obj, "parameters"):
        return np.concatenate([p.detach().cpu().numpy().ravel() for p in obj.parameters()]).astype(np.float32)
    return np.asarray(obj, np.float32)
