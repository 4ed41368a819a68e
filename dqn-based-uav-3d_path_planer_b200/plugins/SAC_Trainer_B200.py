"""Trainer plug-in: SAC (Trainer/SAC_Trainer.py) on the H100 library -- continuous actions (IS_Continuous = 1, the trainer
config/Trainer.xml ships) or discrete ones (IS_Continuous = 0 with PolicyNet_SAC / QValueNet_SAC, the 27-action step).
Constructor takes the reference's parsed Trainer.xml dict (actor / critic / SAC_param sub-dicts)."""
import os

import numpy as np
import torch

import uavrl_b200  # noqa: F401  (repository root must be on sys.path)
from uavrl_b200 import engine
from uavrl_b200.plugins import checkpoint
from uavrl_b200.plugins.xmlconfig import None2Value


class SAC_Trainer_B200:
    ROLE_FILES = ("actor", "critic_1", "critic_2")          # SAC_Trainer.save (:109-119): <role>_SAC_<name>.pth

    def __init__(self, param: dict) -> None:
        actor, critic, sp = param.get('actor'), param.get('critic'), param.get('SAC_param')
        self.IS_Continuous = int(sp.get('IS_Continuous'))
        if self.IS_Continuous not in (0, 1):
            raise ValueError("IS_Continuous must be 1 (continuous actions) or 0 (discrete actions)")
        nets = ('PolicyNetContinuous_SAC', 'QValueNetContinuous_SAC') if self.IS_Continuous else ('PolicyNet_SAC', 'QValueNet_SAC')
        if (actor.get('NetWork'), critic.get('NetWork')) != nets:
            raise ValueError("SAC_Trainer_B200 with IS_Continuous = %d needs %s / %s" % (self.IS_Continuous, nets[0], nets[1]))
        self.name = param.get('name')
        self.replay_size = int(None2Value(param.get('replay_size'), 1000))
        self.Batch_Size = int(None2Value(param.get('Batch_Size'), 128))
        self.save_loop = int(None2Value(param.get('save_loop'), 10))
        self.Is_Train = int(None2Value(param.get('Is_Train'), 1))
        self.IsPriority_Replay = int(None2Value(param.get('IsPriority_Replay'), 0))
        if self.IsPriority_Replay and not self.IS_Continuous:
            raise ValueError("prioritised replay is not available with IS_Continuous = 0: the reference's discrete update() takes "
                             "no importance weights")
        self.w, self.hidden, self.act_dim = int(actor.get('w')), int(actor.get('hiden_dim')), int(actor.get('output'))
        self.lockstep_envs = int(None2Value(param.get('lockstep_envs'), 0))
        if self.IsPriority_Replay and self.lockstep_envs == 0:
            raise ValueError("prioritised replay with SAC needs the lockstep ring (lockstep_envs > 0): its SumTrees index the ring's slots")
        self.device_index = int(None2Value(param.get('device'), 0))
        # n_trainers = G > 1: one independent SAC trainer per block of lockstep_envs / G UAVs (the reference's SAC_Trainer per UAV,
        # PathPlan_City.py:59-69), each with its own replay_size transitions; trainer g is named UAV_<g * lockstep_envs / G>
        # (first_trainer: the global index of trainer 0 when the env plug-in shards the trainers over ranks)
        self.n_trainers = int(None2Value(param.get('n_trainers'), 1))
        G = self.n_trainers
        self.names = checkpoint.trainer_names(self.name, self.lockstep_envs, G, param.get('first_trainer'))
        self._learner = engine.SacLearner(
            self.w, self.hidden, self.act_dim, float(None2Value(actor.get('action_bound'), 1.0)), float(actor.get('lr')),
            float(critic.get('lr')), float(sp.get('alpha_lr')), float(sp.get('target_entropy')), float(sp.get('gamma')),
            float(sp.get('tau')), batch_size=self.Batch_Size, replay_capacity=self.replay_size * G, lockstep_envs=self.lockstep_envs,
            seed=int(None2Value(param.get('seed'), 42)), device=self.device_index, trainers=G, discrete=not self.IS_Continuous)
        self._learner.init_params(int(None2Value(param.get('seed'), 42)))
        if self.IsPriority_Replay:
            # ReplayTree constants (replay_buffer.py:141-148), one tree per trainer as each reference Trainer owns its ReplayTree;
            # the lockstep loop (engine.sac_train_run) then trains on prioritised samples
            self._learner.per_enable()
        self._dev = self._learner.device
        self._losses = torch.zeros(4 * G, device=self._dev)
        self.loss = 0
        self._dist, self._rank, self._world = None, 0, 1
        self.model_dir = None2Value(param.get('model_path'), None)
        self.Load_Mod()

    @property
    def epoch(self):
        return self._learner.scalars()["epoch"]

    @property
    def log_alpha(self):
        return self._learner.scalars()["log_alpha"]

    def get_action(self, state, eps=0.0):
        """SAC_Trainer.get_action (:444-454): [a0, a1] for one state, or an [N, 2] array for a batch (with several trainers the
        [num_UAV, obs] batch: row block g goes to trainer g).  IS_Continuous = 0: an int action index for one state, or an
        [N] int32 array -- a draw from Categorical(actor(s)); eps is ignored, as the reference ignores it."""
        s = np.ascontiguousarray(state, np.float32)
        single = s.ndim == 1
        if single and self.n_trainers > 1:
            raise ValueError("get_action with %d trainers takes the [num_UAV, %d] batch, not one state" % (self.n_trainers, self.w))
        a = self._learner.act(torch.from_numpy(s.reshape(-1, self.w)).to(self._dev)).cpu().numpy()
        if not self.IS_Continuous:
            return int(a[0]) if single else a
        return a[0].tolist() if single else a

    def attach_dist(self, dist, rank, world):
        """Data-parallel training, one process per GPU, each with its own batches: with world > 1, update() sums both critics'
        gradients and squared-error sums over the ranks (dist.all_reduce), steps the critics, then does the same for the
        actor's gradient, loss and entropy sums; every rank's networks, moments and alpha stay bit-identical.  The losses
        average over the global batch (this rank's rows x world)."""
        self._dist, self._rank, self._world = dist, int(rank), int(world)
        if self._world > 1:
            self._xvec = (self._learner.exchange_tensor(0), self._learner.exchange_tensor(1))

    def update(self, transition_dict):
        """SAC_Trainer.update (:317-441) on the batch in transition_dict: the continuous branch, or with IS_Continuous = 0 the
        discrete one (int action indices in 'actions')."""
        states = transition_dict['states']
        if all(len(sub) == 0 for sub in states) if isinstance(states, list) else len(states) == 0:      # :322-324
            sc = self._learner.scalars()
            self._set_counters(sc["epoch"] + 1, sc["adam_step"])
            return {'sum_epoch': self.epoch, 'loss': self.loss}
        dev = self._dev
        f = lambda x, shape: torch.as_tensor(np.asarray(x, np.float32).reshape(shape)).to(dev)  # noqa: E731
        s = f(states, (-1, self.w)); s2 = f(transition_dict['next_states'], (-1, self.w))
        if self.IS_Continuous:
            a = f(transition_dict['actions'], (-1, self.act_dim))
        else:
            a = torch.as_tensor(np.asarray(transition_dict['actions']).astype(np.int32).reshape(-1)).to(dev)
        r = f(transition_dict['rewards'], (-1,)); d = f(transition_dict['dones'], (-1,))
        wts, idx = transition_dict.get('weights'), transition_dict.get('idx')
        if wts is not None:
            if self._world > 1:
                raise ValueError("a weighted (prioritised-replay) update has no split data-parallel form: train with world = 1")
            # importance weights in the critic losses, then ReplayTree.batch_update(tree_idx, e_b) (SAC_Trainer.py:336-352)
            w = f(wts, (-1,))
            ae = torch.zeros(s.shape[0], dtype=torch.float32, device=dev)
            self._learner.update_batch_per(s, a, r, s2, d, w, ae, None, None, self._losses)
            if idx is not None:
                slots = np.asarray(idx, np.int64).reshape(-1) - (self._learner.tree_slots() - 1)
                shape = (-1,) if self.n_trainers == 1 else (self.n_trainers, -1)
                self._learner.per_set_errors(torch.as_tensor(slots.astype(np.int32).reshape(shape)).to(dev), ae.reshape(shape), clip=True)
        elif self._world > 1:
            if not self.IS_Continuous:
                raise ValueError("the data-parallel update is not available with IS_Continuous = 0: train with world = 1")
            L, dist = self._learner, self._dist
            L.critic_grads(s.shape[0] * self._world, batch=(s, a, r, s2, d))
            dist.all_reduce(self._xvec[0], op=dist.ReduceOp.SUM)
            L.apply_critic_grads()
            L.actor_grads()
            dist.all_reduce(self._xvec[1], op=dist.ReduceOp.SUM)
            L.apply_actor_grads(self._losses)
        else:
            self._learner.update_batch(s, a, r, s2, d, None, None, self._losses)
        self.loss = self._losses[0::4]                           # every trainer's actor loss (one trainer: a 1-element tensor)
        if self.save_loop > 0 and self.epoch % self.save_loop == 0:
            self.save()
        return {'sum_epoch': self.epoch, 'loss': self.loss}

    # ---- checkpoints in the reference's format: {'model', 'optimizer', 'epoch'} per network and trainer
    def _rows(self, role):
        """Role `role` of every trainer, (G, P), in ONE device read."""
        return self._learner.get_params(role).reshape(self.n_trainers, -1)

    def _paths(self, directory, g):
        return [os.path.join(directory, '%s_SAC_%s.pth' % (nm, self.names[g])) for nm in self.ROLE_FILES]

    def save(self, directory=None):
        """actor_ / critic_1_ / critic_2_SAC_<name>.pth per trainer (SAC_Trainer.save, :109-119).  Each of the nine vectors
        (three networks, their two Adam moments) is read from the device once for all trainers."""
        directory = directory or self.model_dir or os.path.join(os.getcwd(), 'Mod')
        os.makedirs(directory, exist_ok=True)
        lrs = (self._learner.cfg.actor_lr, self._learner.cfg.critic_lr, self._learner.cfg.critic_lr)
        p, m, v = ([self._rows(base + role) for role in range(3)] for base in (0, 5, 8))
        sc = self._learner.scalars()
        epoch, t = sc["epoch"], sc["adam_step"]
        for g in range(self.n_trainers):
            for role, path in enumerate(self._paths(directory, g)):
                lay = self._learner.layout(role)
                torch.save({'model': checkpoint.model_dict(lay, p[role][g]),
                            'optimizer': checkpoint.adam_dict(lay, m[role][g], v[role][g], t, lrs[role]), 'epoch': epoch}, path)

    def Load_Mod(self, Mod=None):
        """SAC_Trainer.Load_Mod (:70-106): resume actor / critics (+ their Adam moments) of every trainer whose three files
        exist; targets copy the critics.  Every file is parsed into host arrays before anything touches the device; a trainer
        whose files do not parse is left as it is.  Each vector then moves between host and device once for all trainers."""
        directory = self.model_dir or os.path.join(os.getcwd(), 'Mod')
        epoch, step, staged = None, None, {}
        for g in range(self.n_trainers):
            paths = self._paths(directory, g)
            if not all(os.path.exists(p) for p in paths):
                continue
            try:
                mine = [checkpoint.read(p, self._learner.layout(role)) for role, p in enumerate(paths)]
            except Exception as e:          # the reference prints and carries on (SAC_Trainer.py:105-106); nothing was applied
                print(e.args)
                continue
            staged[g], epoch = mine, mine[-1][4]
            for _, m, _, st, _ in mine:     # the last network with optimizer state sets the Adam step
                step = st if m is not None else step
        if not staged:
            return
        rows = {r: self._rows(r) for r in (0, 1, 2, 5, 6, 7, 8, 9, 10)}
        for g, mine in staged.items():
            for role, (flat, m, v, _, _) in enumerate(mine):
                rows[role][g] = flat
                if m is not None:
                    rows[5 + role][g], rows[8 + role][g] = m, v
        for r in (0, 1, 2, 5, 6, 7, 8, 9, 10):
            self._learner.set_params(r, rows[r])
        for r in (1, 2):
            self._learner.set_params(r + 2, rows[r])
        self._set_counters(epoch, 0 if step is None else step)

    def _set_counters(self, epoch, adam_step):
        """epoch and Adam step; every trainer keeps its own alpha (set_scalars alone would give all of them trainer 0's)."""
        al = self._learner.alpha()
        self._learner.set_scalars(*(float(x) for x in al[0]), epoch, adam_step)
        self._learner.set_alpha(al)

    def hard_update(self):
        pass

    def _learner_reset_lockstep(self):
        pass
