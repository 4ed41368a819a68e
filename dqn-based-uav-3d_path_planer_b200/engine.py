"""Thin object layer over the C ABI (include/uavrl.h): EnvBatch and Learner.

torch is used here only for device memory, streams and (elsewhere) torch.distributed; every
computation on the hot path happens inside libuavrl_b200.so.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import (ACT_CONT_F32, ACT_CONT_F64, ACT_DISCRETE27, ALGO_DDQN, ALGO_DQN, ALGO_DUELING,  # noqa: F401
                   INFO_NAMES, OBS_DIM, UavrlError, check)


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        return C.c_void_p(t.data_ptr())
    if isinstance(t, np.ndarray):
        return C.c_void_p(t.ctypes.data)
    raise TypeError(type(t))


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class City:
    """Box dims + cylinder table [n,5] = cx, cy, cz, _R, _H (config/buildings.xml)."""

    def __init__(self, length, width, h, buildings):
        self.len, self.width, self.h = float(length), float(width), float(h)
        self.buildings = np.ascontiguousarray(buildings, np.float64).reshape(-1, 5)


class UavParams:
    """config/UAV.xml fields the step uses (Agents/UAV.py:25-32)."""

    def __init__(self, max_v=1.0, min_v=0.6, steering=np.pi / 6, climb_rate=1.0, max_step=150):
        self.max_v, self.min_v, self.steering = float(max_v), float(min_v), float(steering)
        self.climb_rate, self.max_step = float(climb_rate), int(max_step)


class EnvBatch:
    """N UAV environments stepped in lockstep on one GPU."""

    def __init__(self, city, params, n_envs, max_subgoals=64, device=0, auto_reset=False):
        self.city, self.params, self.n, self.K = city, params, int(n_envs), int(max_subgoals)
        self.device = torch.device("cuda", device)
        self.cfg = _lib.EnvConfig()
        c = self.cfg
        c.n_envs, c.max_subgoals = self.n, self.K
        c.len, c.width, c.h = city.len, city.width, city.h
        c.max_v, c.min_v, c.steering_angle = params.max_v, params.min_v, params.steering
        c.max_step, c.climb_rate = params.max_step, params.climb_rate
        c.n_buildings = city.buildings.shape[0]
        c.buildings_host = city.buildings.ctypes.data_as(C.POINTER(C.c_double))
        c.device, c.auto_reset = device, int(bool(auto_reset))
        self.h = C.c_void_p()
        check(_lib.lib().uavrl_env_create(C.byref(c), C.byref(self.h)))

    def close(self):
        if self.h:
            _lib.lib().uavrl_env_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- scenarios
    def make_scenarios(self, n, seed=42, rrt_step=30):
        """Host-side reset draws + RRT (UAV.py:344-360, RRT.py:63-105); returns the pool arrays."""
        start = np.zeros((n, 3)); goal = np.zeros((n, 3)); heading = np.zeros(n)
        sub = np.zeros((n, self.K, 3)); n_sub = np.zeros(n, np.int32)
        check(_lib.lib().uavrl_make_scenarios(C.byref(self.cfg), C.c_uint64(seed), n, rrt_step, _ptr(start),
                                              _ptr(goal), _ptr(heading), _ptr(sub), _ptr(n_sub)))
        return dict(start=start, goal=goal, heading=heading, sub=sub, n_sub=n_sub)

    def set_pool(self, start, goal, heading, sub, n_sub, alias0=None):
        start = np.ascontiguousarray(start, np.float64).reshape(-1, 3)
        P = start.shape[0]
        goal = np.ascontiguousarray(goal, np.float64).reshape(P, 3)
        heading = np.ascontiguousarray(heading, np.float64).reshape(P)
        sub_in = np.asarray(sub, np.float64)
        subp = np.zeros((P, self.K, 3), np.float64)
        subp[:, :sub_in.shape[1], :] = sub_in
        n_sub = np.ascontiguousarray(n_sub, np.int32).reshape(P)
        al = None if alias0 is None else np.ascontiguousarray(alias0, np.uint8).reshape(P)
        check(_lib.lib().uavrl_env_set_pool(self.h, P, _ptr(start), _ptr(goal), _ptr(heading), _ptr(subp),
                                            _ptr(n_sub), _ptr(al)))
        self.pool_size = P

    def generate_pool(self, n, seed=42, rrt_step=30):
        """Reset draws + RRT on the device, straight into the env's pool (same scenarios as make_scenarios + set_pool)."""
        check(_lib.lib().uavrl_env_generate_pool(self.h, int(n), C.c_uint64(seed), int(rrt_step), _stream(self.device)))
        self.pool_size = int(n)

    def get_pool(self):
        P = self.pool_size
        start = np.zeros((P, 3)); goal = np.zeros((P, 3)); v0 = np.zeros((P, 3))
        sub = np.zeros((P, self.K, 3)); n_sub = np.zeros(P, np.int32)
        check(_lib.lib().uavrl_env_get_pool(self.h, _ptr(start), _ptr(goal), _ptr(v0), _ptr(sub), _ptr(n_sub)))
        return dict(start=start, goal=goal, v0=v0, sub=sub, n_sub=n_sub)

    def reset(self, first_scenario=0):
        check(_lib.lib().uavrl_env_reset(self.h, int(first_scenario), _stream(self.device)))

    # -- stepping (device buffers)
    def observe(self, out=None):
        if out is None:
            out = torch.empty((self.n, OBS_DIM), dtype=torch.float32, device=self.device)
        check(_lib.lib().uavrl_env_observe(self.h, _ptr(out), _stream(self.device)))
        return out

    def step(self, actions, kind=None, out=None):
        """actions: cuda tensor, float32/float64 (continuous a0) or int32 (discrete-27 index)."""
        if kind is None:
            kind = {torch.float32: ACT_CONT_F32, torch.float64: ACT_CONT_F64, torch.int32: ACT_DISCRETE27}[actions.dtype]
        if out is None:
            dev = self.device
            out = dict(obs=torch.empty((self.n, OBS_DIM), dtype=torch.float32, device=dev),
                       reward=torch.empty(self.n, dtype=torch.float32, device=dev),
                       done=torch.empty(self.n, dtype=torch.uint8, device=dev),
                       info=torch.empty(self.n, dtype=torch.uint8, device=dev),
                       collision=torch.empty(self.n, dtype=torch.uint8, device=dev),
                       ended=torch.empty(self.n, dtype=torch.uint8, device=dev))
        check(_lib.lib().uavrl_env_step(self.h, kind, _ptr(actions), _ptr(out.get("obs")), _ptr(out.get("reward")),
                                        _ptr(out.get("done")), _ptr(out.get("info")), _ptr(out.get("collision")),
                                        _ptr(out.get("ended")), _stream(self.device)))
        return out

    def step_host(self, actions, kind, obs, reward, done, info=None, collision=None, ended=None):
        """Host-buffer entry point (numpy arrays or pinned CPU tensors): H2D + step + D2H + sync."""
        check(_lib.lib().uavrl_env_step_host(self.h, kind, _ptr(actions), _ptr(obs), _ptr(reward), _ptr(done),
                                             _ptr(info), _ptr(collision), _ptr(ended)))

    def get_state(self):
        n = self.n
        out = {k: np.zeros(n, np.float64) for k in
               ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len", "reward64")}
        out.update({k: np.zeros(n, np.int32) for k in ("step", "cursor", "scenario")})
        out["done"] = np.zeros(n, np.uint8)
        st = _lib.EnvStateHost()
        for k, v in out.items():
            ct = {np.dtype(np.float64): C.c_double, np.dtype(np.int32): C.c_int32, np.dtype(np.uint8): C.c_uint8}[v.dtype]
            setattr(st, k, v.ctypes.data_as(C.POINTER(ct)))
        check(_lib.lib().uavrl_env_get_state(self.h, C.byref(st)))
        return out

    def set_state(self, **arrays):
        """Overwrite per-UAV state (px, py, pz, vx, vy, V, score, total_score, path_len: float64; step: int32; done: uint8)."""
        st = _lib.EnvStateHost()
        keep = []
        for k, v in arrays.items():
            if k in ("step",):
                a, ct = np.ascontiguousarray(v, np.int32), C.c_int32
            elif k == "done":
                a, ct = np.ascontiguousarray(v, np.uint8), C.c_uint8
            elif k in ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len"):
                a, ct = np.ascontiguousarray(v, np.float64), C.c_double
            else:
                raise KeyError(k)
            assert a.shape == (self.n,), (k, a.shape)
            keep.append(a)
            setattr(st, k, a.ctypes.data_as(C.POINTER(ct)))
        check(_lib.lib().uavrl_env_set_state(self.h, C.byref(st)))

    # -- optional models (uavrl_env_set_extras): energy accumulator, moving-obstacle APF, trajectory recording
    def set_extras(self, power=None, obstacle_v=None, track_envs=0, track_capacity=0):
        """power: dict P_i, v_0, d_0, rho, s, A, P_b, F_b, xi (config/UAV.xml <Fly_power>; xi = 0.8 + 0.02 j) -> per-UAV energy;
        obstacle_v: [n_buildings, 3] obstacle velocities -> APF_Enabled behaviour (UAV.py:156-210, 448-453);
        track_envs / track_capacity: record UAV.path of the first track_envs UAVs.  Call before reset()."""
        x = _lib.EnvExtras()
        if power is not None:
            x.energy_enabled = 1
            for k in ("P_i", "v_0", "d_0", "rho", "s", "A", "P_b", "F_b", "xi"):
                setattr(x, k, float(power[k]))
        keep = None
        if obstacle_v is not None:
            keep = np.ascontiguousarray(obstacle_v, np.float64).reshape(-1, 3)
            assert keep.shape[0] == self.city.buildings.shape[0]
            x.apf_enabled = 1
            x.obstacle_v_host = keep.ctypes.data_as(C.POINTER(C.c_double))
        x.track_envs, x.track_capacity = int(track_envs), int(track_capacity)
        check(_lib.lib().uavrl_env_set_extras(self.h, C.byref(x)))
        self._track_cap = int(track_capacity)

    def get_energy(self):
        out = np.zeros(self.n, np.float64)
        check(_lib.lib().uavrl_env_get_energy(self.h, _ptr(out)))
        return out

    def get_energy_total(self):
        t = C.c_double()
        check(_lib.lib().uavrl_env_get_energy_total(self.h, C.byref(t)))
        return t.value

    def get_path(self, e, which=0):
        """UAV.path of tracked UAV e: which = 0 the episode in progress, 1 the last finished episode -> [n, 3]."""
        buf = np.zeros((self._track_cap, 3), np.float64)
        n = C.c_int32()
        check(_lib.lib().uavrl_env_get_path(self.h, int(e), int(which), self._track_cap, _ptr(buf), C.byref(n)))
        return buf[:min(n.value, self._track_cap)].copy()

    def get_subgoals(self):
        out = np.zeros((self.n, self.K, 3), np.float64)
        check(_lib.lib().uavrl_env_get_subgoals(self.h, _ptr(out)))
        return out

    def threaten_rate(self, pts):
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        out = np.zeros(pts.shape[0], np.uint8)
        check(_lib.lib().uavrl_env_threaten_rate(self.h, pts.shape[0], _ptr(pts), _ptr(out)))
        return out


NET_KINDS = {                       # BaseClass/BaseCNN.py class name -> (hidden widths as f(h), dueling)
    "Qnet2": (lambda h: [h], 0),
    "QValueNet_SAC": (lambda h: [h, h], 0),
    "VAnet2": (lambda h: [h], 1),
    "VAnet3": (lambda h: [2 * h, h], 1),
    "VAnet4": (lambda h: [2 * h, h, h], 1),
    "VAnet5": (lambda h: [2 * h, h, h, h], 1),
}


def _linears(*layers):
    """Layout of torch.nn.Linear layers given as (name, out, in): a list of (state_dict key, shape)."""
    return [(k, s) for nm, o, i in layers for k, s in ((nm + ".weight", (o, i)), (nm + ".bias", (o,)))]


def _size(layout):
    return sum(int(np.prod(s)) for _, s in layout)


def init_draw(layout, gen):
    """torch.nn.Linear default init (kaiming_uniform(a=sqrt(5)) == U(+-1/sqrt(fan_in)) for W and b) of every tensor of a
    layout, in order, from torch generator `gen`: the flat float32 parameters."""
    parts = []
    for _, shape in layout:
        if len(shape) == 2:                 # a weight; its bias follows and shares the fan-in
            bound = 1.0 / np.sqrt(shape[1])
        parts.append((torch.rand(int(np.prod(shape)), generator=gen) * 2 - 1) * bound)
    return torch.cat(parts).numpy()


class Learner:
    """Q-network + Adam + replay on one GPU (DQN / DDQN / DuelingDQN trainers of the reference).

    trainers = G > 1: G independent trainers of this network in one handle (one Trainer per UAV group, PathPlan_City.py:59-69).
    The lockstep envs split into G blocks of lockstep_envs / G, trainer g learns from its block only and computes what a
    stand-alone Learner(seed=seed + g, replay_capacity=replay_capacity // G, lockstep_envs=lockstep_envs // G) computes.
    Parameters are then (G, P) arrays, act / update_batch take G equal row blocks and loss tensors are [G]
    (include/uavrl.h, uavrl_learner_create_trainers)."""

    def __init__(self, in_dim=OBS_DIM, hidden=(64, 64), n_actions=27, dueling=False, algo=ALGO_DDQN, lr=5e-4,
                 gamma=0.99, batch_size=64, update_loop=3, replay_capacity=10000, lockstep_envs=0, seed=42, device=0, loss="mse",
                 trainers=1):
        self.device = torch.device("cuda", device)
        c = _lib.LearnerConfig()
        c.loss_kind = {"mse": 0, "huber": 1}[loss]
        c.in_dim, c.n_hidden, c.n_actions, c.dueling, c.algo = in_dim, len(hidden), n_actions, int(dueling), algo
        for i, h in enumerate(hidden):
            c.hidden[i] = int(h)
        c.lr, c.gamma, c.batch_size, c.update_loop = lr, gamma, batch_size, update_loop
        c.replay_capacity, c.lockstep_envs, c.seed, c.device = replay_capacity, lockstep_envs, seed, device
        self.cfg = c
        self.in_dim, self.hidden, self.n_actions, self.dueling = in_dim, list(hidden), n_actions, bool(dueling)
        self.h = C.c_void_p()
        check(_lib.lib().uavrl_learner_create_trainers(C.byref(c), int(trainers), C.byref(self.h)))
        self.P = int(_lib.lib().uavrl_learner_param_count(self.h))
        self.G = int(_lib.lib().uavrl_learner_trainer_count(self.h))
        assert _size(self.layout()) == self.P, (self.layout(), self.P)

    def layout(self):
        """(state_dict key, shape) of every tensor in flat-parameter order, named as the reference's networks
        (BaseClass/BaseCNN.py) name them: fc1 .. fcN, then fc_A and fc_V for a dueling head."""
        ins = [self.in_dim] + self.hidden
        trunk = [("fc%d" % (i + 1), w, ins[i]) for i, w in enumerate(self.hidden)]
        if self.dueling:
            return _linears(*trunk, ("fc_A", self.n_actions, ins[-1]), ("fc_V", 1, ins[-1]))
        return _linears(*trunk, ("fc%d" % len(ins), self.n_actions, ins[-1]))

    def close(self):
        if self.h:
            _lib.lib().uavrl_learner_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- parameters (flat, state_dict order)
    def init_params(self, seed=0):
        """torch.nn.Linear default init (kaiming_uniform(a=sqrt(5)) == U(+-1/sqrt(fan_in)) for W and b),
        independent draws for q_local and q_target like the reference's two Create_Network calls.
        Trainer g of a grouped learner draws with seed + g."""
        gens = [torch.Generator().manual_seed(seed + g) for g in range(self.G)]
        draws = [[init_draw(self.layout(), gen) for _ in (0, 1)] for gen in gens]
        for which in (0, 1):
            self.set_params(np.stack([d[which] for d in draws]), which)

    def _param_shape(self):
        return (self.P,) if self.G == 1 else (self.G, self.P)

    def set_params(self, flat, which=0):
        """which: 0 q_local, 1 q_target, 2 / 3 Adam exp_avg / exp_avg_sq, 4 gradient; (P,) or, with trainers > 1, (G, P)."""
        flat = np.ascontiguousarray(flat, np.float32)
        assert flat.size == self.G * self.P, (flat.shape, self._param_shape())
        check(_lib.lib().uavrl_learner_set_params(self.h, which, _ptr(flat)))

    def get_params(self, which=0):
        out = np.zeros(self._param_shape(), np.float32)
        check(_lib.lib().uavrl_learner_get_params(self.h, which, _ptr(out)))
        return out

    def trainer_count(self):
        return self.G

    def counters(self):
        e, t = C.c_int64(), C.c_int64()
        check(_lib.lib().uavrl_learner_get_counters(self.h, C.byref(e), C.byref(t)))
        return e.value, t.value

    def set_counters(self, epoch, adam_step):
        check(_lib.lib().uavrl_learner_set_counters(self.h, int(epoch), int(adam_step)))

    # -- acting / replay / update
    def act(self, obs, eps, is_train=True, u_tape=None, rand_tape=None, want_q=False):
        n = obs.shape[0]
        a = torch.empty(n, dtype=torch.int32, device=self.device)
        q = torch.empty((n, self.n_actions), dtype=torch.float32, device=self.device) if want_q else None
        check(_lib.lib().uavrl_learner_act(self.h, _ptr(obs), n, float(eps), int(is_train), _ptr(u_tape),
                                           _ptr(rand_tape), _ptr(a), _ptr(q), _stream(self.device)))
        return (a, q) if want_q else a

    def push(self, obs, act, rew, next_obs, done):
        check(_lib.lib().uavrl_replay_push(self.h, obs.shape[0], _ptr(obs), _ptr(act), _ptr(rew), _ptr(next_obs),
                                           _ptr(done), _stream(self.device)))

    def replay_size(self):
        return int(_lib.lib().uavrl_replay_size(self.h))

    def gather(self, logical_idx):
        idx = np.ascontiguousarray(logical_idx, np.int64)
        n = idx.size
        s = np.zeros((n, self.in_dim), np.float32); s2 = np.zeros((n, self.in_dim), np.float32)
        a = np.zeros(n, np.int32); r = np.zeros(n, np.float32); d = np.zeros(n, np.uint8)
        check(_lib.lib().uavrl_replay_gather(self.h, n, _ptr(idx), _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d)))
        return s, a, r, s2, d

    def _loss(self, loss):
        """A caller's loss tensor: the update writes one loss per trainer, so it must hold at least G floats."""
        if loss is not None and loss.numel() < self.G:
            raise ValueError("loss holds %d elements; a learner with %d trainers writes %d losses" % (loss.numel(), self.G, self.G))
        return _ptr(loss)

    def update(self, idx_tape=None, loss=None):
        check(_lib.lib().uavrl_learner_update(self.h, _ptr(idx_tape), self._loss(loss), _stream(self.device)))

    def federate(self, probe_states=None, probe_tape=None, want_details=False):
        """Selective federated aggregation across the trainers (PathPlan_City.Federated_Learning_choice, include/uavrl.h
        uavrl_learner_federate).  probe_states: (G, 10, in_dim) device tensor, or None to draw the probes from the lockstep
        ring; probe_tape: (G, 10) trainer-local replay indices for the ring draw, a host array (checked, then uploaded) or a
        device int32 tensor.  want_details: returns device tensors (probe_idx (G, 10), losses (G, G), chosen (G, max(1, k)))."""
        G = self.G
        if probe_tape is not None and not isinstance(probe_tape, torch.Tensor):
            tape = np.ascontiguousarray(probe_tape, np.int64)
            if tape.shape != (G, 10):
                raise ValueError("probe_tape must be (%d, 10), got %s" % (G, tape.shape))
            if any(len(set(row.tolist())) != 10 for row in tape):
                raise ValueError("probe_tape rows must hold 10 distinct indices")
            n_g = self.replay_size() // G
            if (tape < 0).any() or (tape >= n_g).any():
                raise ValueError("probe_tape indices must lie in [0, %d) (transitions per trainer)" % n_g)
            probe_tape = torch.from_numpy(tape.astype(np.int32)).to(self.device)
        if probe_states is not None and tuple(probe_states.shape) != (G, 10, self.in_dim):
            raise ValueError("probe_states must be (%d, 10, %d)" % (G, self.in_dim))
        k = (G - 1) // 2
        idx = losses = chosen = None
        if want_details:
            idx = torch.empty((G, 10), dtype=torch.int32, device=self.device)
            losses = torch.empty((G, G), dtype=torch.float32, device=self.device)
            chosen = torch.empty((G, max(1, k)), dtype=torch.int32, device=self.device)
        check(_lib.lib().uavrl_learner_federate(self.h, _ptr(probe_states), _ptr(probe_tape), _ptr(idx), _ptr(losses), _ptr(chosen),
                                                _stream(self.device)))
        if want_details:
            return idx, losses, chosen

    def update_batch(self, s, a, r, s2, d, loss=None):
        check(_lib.lib().uavrl_learner_update_batch(self.h, s.shape[0], _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d),
                                                    self._loss(loss), _stream(self.device)))

    def update_batch_per(self, s, a, r, s2, d, is_weights=None, abs_err_out=None, loss=None):
        """update_batch with per-sample importance weights in the loss and |Q - y| written back (prioritised replay)."""
        check(_lib.lib().uavrl_learner_update_batch_per(self.h, s.shape[0], _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d),
                                                        _ptr(is_weights), _ptr(abs_err_out), _ptr(loss), _stream(self.device)))

    # -- prioritised replay (SumTree + ReplayTree of the reference, BaseClass/replay_buffer.py:57-223)
    def per_enable(self, alpha=-1.0, beta0=-1.0, beta_inc=-1.0, eps=-1.0, err_upper=-1.0):
        check(_lib.lib().uavrl_per_enable(self.h, alpha, beta0, beta_inc, eps, err_upper))
        self.per_slots = int(self.cfg.replay_capacity) if not self.cfg.lockstep_envs else None

    def per_enable_trainers(self, alpha=-1.0, beta0=-1.0, beta_inc=-1.0, eps=-1.0, err_upper=-1.0):
        """Prioritised replay with one tree per trainer (include/uavrl.h uavrl_per_enable_trainers); per_enable when G = 1.
        With G > 1 the per_* methods then take and return (G, ...) arrays of trainer-local slots."""
        check(_lib.lib().uavrl_per_enable_trainers(self.h, alpha, beta0, beta_inc, eps, err_upper))
        self.per_slots = int(self.cfg.replay_capacity) if not self.cfg.lockstep_envs else None

    def _per_shape(self, n):
        return (n,) if self.G == 1 else (self.G, n)

    def per_sample(self, batch, u_tape=None):
        """ReplayTree.sample2: (slots int32 [B], importance weights float32 [B]) on the device; (G, B) each on a grouped
        learner, u_tape (G, B)."""
        slots = torch.empty(self._per_shape(batch), dtype=torch.int32, device=self.device)
        w = torch.empty(self._per_shape(batch), dtype=torch.float32, device=self.device)
        check(_lib.lib().uavrl_per_sample(self.h, int(batch), _ptr(u_tape), _ptr(slots), _ptr(w), _stream(self.device)))
        return slots, w

    def _per_n(self, slots):
        """Slots per trainer of a (n,) or, grouped, (G, n) slot array."""
        if self.G > 1 and (slots.dim() != 2 or slots.shape[0] != self.G):
            raise ValueError("a learner with %d trainers takes (%d, n) slots, got %s" % (self.G, self.G, tuple(slots.shape)))
        return int(slots.shape[-1])

    def per_set_errors(self, slots, abs_err, clip=True):
        check(_lib.lib().uavrl_per_set_errors(self.h, self._per_n(slots), _ptr(slots), _ptr(abs_err), int(bool(clip)),
                                              _stream(self.device)))

    def per_set_priorities(self, slots, priorities):
        check(_lib.lib().uavrl_per_set_priorities(self.h, self._per_n(slots), _ptr(slots), _ptr(priorities), _stream(self.device)))

    def per_state(self, n_slots):
        """(leaves, total, beta); grouped: n_slots per trainer, leaves (G, n_slots) and totals (G,)."""
        leaves = np.zeros(self._per_shape(int(n_slots)), np.float64)
        totals, beta = np.zeros(self.G, np.float64), C.c_double()
        check(_lib.lib().uavrl_per_get(self.h, _ptr(leaves), totals.ctypes.data_as(C.POINTER(C.c_double)), C.byref(beta)))
        return leaves, (float(totals[0]) if self.G == 1 else totals), beta.value

    def compute_grads(self, global_batch, idx_tape=None, loss=None):
        check(_lib.lib().uavrl_learner_compute_grads(self.h, _ptr(idx_tape), int(global_batch), _ptr(loss),
                                                     _stream(self.device)))

    def grad_tensor(self):
        """The device gradient vector as a torch view (for torch.distributed.all_reduce)."""
        ptr = _lib.lib().uavrl_learner_grad_ptr(self.h)
        arr = (C.c_float * self.P).from_address(ptr) if False else None  # noqa: F841 (device memory: no host view)
        return _DevView(ptr, self.P, self.device).tensor()

    def connect_peers(self, dist, rank, world):
        """Exchange the CUDA IPC handles of the symmetric gradient receive buffers over torch.distributed and map
        every peer's buffer (NVLink P2P) -- enables update_dp(), the fused one-shot all-reduce + Adam."""
        hg = (C.c_ubyte * 64)()
        check(_lib.lib().uavrl_learner_comm_init(self.h, rank, world, hg, None))
        mine = torch.tensor(list(bytes(hg)), dtype=torch.uint8, device=self.device)
        allh = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(allh, mine)
        g = np.ascontiguousarray(torch.stack(allh).cpu().numpy())
        check(_lib.lib().uavrl_learner_comm_connect(self.h, _ptr(g), None))
        dist.barrier(device_ids=[self.device.index])

    def connect_self(self):
        """world = 1: the data-parallel optimiser kernel (push into the local receive buffer, gather, all-reduce + Adam) on
        one GPU -- the self-test of the fused path that needs no second device."""
        hg = (C.c_ubyte * 64)()
        check(_lib.lib().uavrl_learner_comm_init(self.h, 0, 1, hg, None))
        check(_lib.lib().uavrl_learner_comm_connect(self.h, hg, None))

    def update_dp(self, global_batch, idx_tape=None, loss=None):
        check(_lib.lib().uavrl_learner_update_dp(self.h, _ptr(idx_tape), int(global_batch), _ptr(loss), _stream(self.device)))

    def apply_grads(self):
        check(_lib.lib().uavrl_learner_apply_grads(self.h, _stream(self.device)))

    def hard_update(self):
        check(_lib.lib().uavrl_learner_hard_update(self.h, _stream(self.device)))

    def set_tensor_cores(self, enable):
        """True = wgmma 3xTF32 forward passes (default when the net fits), False = fp32 CUDA cores."""
        return bool(_lib.lib().uavrl_learner_set_tensor_cores(self.h, int(bool(enable))))

    def td_fused(self, batch=None):
        """True when an update of `batch` transitions runs its TD-target pass(es) inside the training kernel."""
        return bool(_lib.lib().uavrl_learner_td_fused(self.h, int(self.cfg.batch_size if batch is None else batch)))

    def route(self, n):
        """Which kernels an act / TD pass over n samples and an update of a batch of n run, with the current
        set_tensor_cores setting: tc_fwd / tc_train = "fixed" (compile-time wgmma chains), "generic" (runtime k-step
        chains) or None (the fp32 CUDA-core kernel); fwd_rows / train_rows = rows per tile of those tensor-core kernels
        (None when not used); td_fused = the TD-target pass(es) run inside the training kernel; fp32_dual = the fp32 update
        kernel keeps both networks' weights in shared memory at once."""
        out = (C.c_int32 * 6)()
        check(_lib.lib().uavrl_learner_tc_route(self.h, int(n), out))
        variant = {0: None, 1: "generic", 2: "fixed"}
        return dict(tc_fwd=variant[out[0]], tc_train=variant[out[1]], fwd_rows=out[2] or None, train_rows=out[3] or None,
                    td_fused=bool(out[4]), fp32_dual=bool(out[5]))

    def lockstep_restart(self):
        check(_lib.lib().uavrl_learner_lockstep_restart(self.h))

    def set_is_train(self, is_train):
        """Trainer.Is_Train for the lockstep loops: False = get_action is always greedy (DuelingDQN_Trainer.py:90)."""
        check(_lib.lib().uavrl_learner_set_is_train(self.h, int(bool(is_train))))


class _DevView:
    """Expose a raw device pointer as a torch tensor through __cuda_array_interface__."""

    def __init__(self, ptr, n, device):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "version": 2}
        self.device = device

    def tensor(self):
        return torch.as_tensor(self, device=self.device)


def train_run(env, learner, n_iters, eps, updates_per_iter=1, do_update=True, want_stats=True):
    """uavrl_train_run: n_iters lockstep iterations of act -> step -> (ring) -> update."""
    st = _lib.TrainStats()
    check(_lib.lib().uavrl_train_run(env.h, learner.h, int(n_iters), float(eps), int(updates_per_iter),
                                     int(bool(do_update)), C.byref(st) if want_stats else None, _stream(env.device)))
    return st


def train_profile(env, learner, n_iters, eps):
    """Per-kernel device time (ms, summed over n_iters) of
    {act, env_step, td_target, fwd_bwd, weight_grad, reduce_adam}."""
    ms = np.zeros(6, np.float32)
    check(_lib.lib().uavrl_train_profile(env.h, learner.h, int(n_iters), float(eps), _ptr(ms), _stream(env.device)))
    return ms


def train_run_dp(env, learner, n_iters, eps, global_batch):
    """uavrl_train_run_dp: lockstep iterations whose update is the fused NVLink all-reduce + Adam."""
    check(_lib.lib().uavrl_train_run_dp(env.h, learner.h, int(n_iters), float(eps), int(global_batch), _stream(env.device)))


class SacLearner:
    """SAC continuous (the reference's shipped trainer, config/Trainer.xml) on one GPU.  obs_dim must be a multiple of 4 in
    [4, 124], hidden in [1, 128], and the networks must fit the kernels' shared memory (sac_smem_bytes).  Parameter roles:
    0-4 actor, critic_1, critic_2 and their targets, 5-7 / 8-10 Adam moments, 11-13 the last reduced gradients (read-only).

    trainers = G > 1: G independent SAC trainers in one handle (one SAC_Trainer per UAV group, PathPlan_City.py:59-69).  The
    lockstep envs split into G blocks of lockstep_envs / G, trainer g learns from its block only and computes what a
    stand-alone SacLearner(seed=seed + g, replay_capacity=replay_capacity // G, lockstep_envs=lockstep_envs // G) computes.
    Parameters are then (G, P) arrays, alpha() is (G, 3), act / update_batch take G equal row blocks and loss tensors hold
    [G][4] floats (include/uavrl.h, uavrl_sac_create_trainers)."""
    ROLES = ("actor", "critic_1", "critic_2", "target_critic_1", "target_critic_2")

    def __init__(self, obs_dim=OBS_DIM, hidden=64, act_dim=2, action_bound=1.0, actor_lr=1e-4, critic_lr=1e-3, alpha_lr=1e-4,
                 target_entropy=1.0, gamma=0.99, tau=0.05, batch_size=64, replay_capacity=10000, lockstep_envs=0, seed=42, device=0,
                 trainers=1):
        self.device = torch.device("cuda", device)
        c = _lib.SacConfig(obs_dim, hidden, act_dim, action_bound, actor_lr, critic_lr, alpha_lr, target_entropy, gamma, tau,
                           batch_size, replay_capacity, lockstep_envs, seed, device)
        self.cfg = c
        self.h = C.c_void_p()
        check(_lib.lib().uavrl_sac_create_trainers(C.byref(c), int(trainers), C.byref(self.h)))
        self.P = [int(_lib.lib().uavrl_sac_param_count(self.h, r)) for r in range(5)]
        self.G = int(_lib.lib().uavrl_sac_trainer_count(self.h))
        assert [_size(self.layout(r)) for r in range(5)] == self.P, self.P

    def layout(self, role):
        """(state_dict key, shape) of every tensor of network `role` in flat-parameter order, named as the reference's
        PolicyNetContinuous_SAC (role 0) and QValueNetContinuous_SAC (roles 1-4: the critics and their targets) name them."""
        o, h, a = self.cfg.obs_dim, self.cfg.hidden, self.cfg.act_dim
        if role == 0:
            return _linears(("fc1", h, o), ("fc_mu", a, h), ("fc_std", a, h))
        return _linears(("fc1", h, o + a), ("fc2", h, h), ("fc_out", a, h))

    def close(self):
        if self.h:
            _lib.lib().uavrl_sac_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _param_shape(self, role):
        n = self.P[role] if role < 5 else self.P[(role - 5) % 3]
        return (n,) if self.G == 1 else (self.G, n)

    def set_params(self, role, flat):
        """(P,) or, with trainers > 1, (G, P) values of `role` for every trainer."""
        flat = np.ascontiguousarray(flat, np.float32)
        shape = self._param_shape(role)
        assert flat.size == int(np.prod(shape)), (flat.shape, shape)
        check(_lib.lib().uavrl_sac_set_params(self.h, role, _ptr(flat)))

    def get_params(self, role):
        out = np.zeros(self._param_shape(role), np.float32)
        check(_lib.lib().uavrl_sac_get_params(self.h, role, _ptr(out)))
        return out

    def trainer_count(self):
        return self.G

    def init_params(self, seed=0):
        """nn.Linear default init for actor and the two critics; targets copy the critics (SAC_Trainer.py:33-34).
        Trainer g of a grouped learner draws with seed + g."""
        gens = [torch.Generator().manual_seed(seed + g) for g in range(self.G)]
        draws = [[init_draw(self.layout(r), gen) for r in range(3)] for gen in gens]
        for r in range(3):
            flat = np.stack([d[r] for d in draws])
            self.set_params(r, flat)
            if r > 0:
                self.set_params(r + 2, flat)

    def alpha(self):
        """Every trainer's (log_alpha, Adam exp_avg, Adam exp_avg_sq): a (G, 3) array."""
        out = np.zeros((self.G, 3), np.float32)
        check(_lib.lib().uavrl_sac_get_alpha(self.h, _ptr(out)))
        return out

    def set_alpha(self, triples):
        t = np.ascontiguousarray(triples, np.float32)
        if t.size != 3 * self.G:
            raise ValueError("alpha triples must be (%d, 3), got %s" % (self.G, t.shape))
        check(_lib.lib().uavrl_sac_set_alpha(self.h, _ptr(t)))

    def federate_actors(self):
        """Federated_Learning_AC (PathPlan_City.py:590-601, include/uavrl.h uavrl_sac_federate_actors): every trainer's actor
        becomes the float32 sum of all G actors (the reference's division by G is lost); nothing else changes."""
        check(_lib.lib().uavrl_sac_federate_actors(self.h, _stream(self.device)))

    def _losses(self, losses):
        """A caller's loss tensor: an update writes 4 losses per trainer, so it must hold at least 4 G floats."""
        if losses is not None and losses.numel() < 4 * self.G:
            raise ValueError("losses holds %d elements; a learner with %d trainers writes %d losses" % (losses.numel(), self.G, 4 * self.G))
        return _ptr(losses)

    def scalars(self):
        la, m, v = C.c_float(), C.c_float(), C.c_float()
        e, t = C.c_int64(), C.c_int64()
        check(_lib.lib().uavrl_sac_get_scalars(self.h, C.byref(la), C.byref(m), C.byref(v), C.byref(e), C.byref(t)))
        return dict(log_alpha=la.value, la_m=m.value, la_v=v.value, epoch=e.value, adam_step=t.value)

    def set_scalars(self, log_alpha, la_m=0.0, la_v=0.0, epoch=0, adam_step=0):
        check(_lib.lib().uavrl_sac_set_scalars(self.h, float(log_alpha), float(la_m), float(la_v), int(epoch), int(adam_step)))

    def act(self, obs, eps=None):
        n = obs.shape[0]
        a = torch.empty((n, self.cfg.act_dim), dtype=torch.float32, device=self.device)
        check(_lib.lib().uavrl_sac_act(self.h, _ptr(obs), n, _ptr(eps), _ptr(a), _stream(self.device)))
        return a

    def update_batch(self, s, a, r, s2, d, eps_next=None, eps_cur=None, losses=None):
        check(_lib.lib().uavrl_sac_update_batch(self.h, s.shape[0], _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d), _ptr(eps_next),
                                                _ptr(eps_cur), self._losses(losses), _stream(self.device)))

    def grads(self, role):
        """The gradient of network `role` (0 actor, 1 critic_1, 2 critic_2) that the last update reduced and fed to Adam."""
        return self.get_params(11 + role)

    def smem_bytes(self):
        """Shared memory per block of the target, critic, actor and get_action kernels (see sac_smem_bytes)."""
        return sac_smem_bytes(self.cfg.obs_dim, self.cfg.hidden, self.cfg.device)

    def replay_size(self):
        return int(_lib.lib().uavrl_sac_replay_size(self.h))

    def gather(self, logical_idx):
        """Transitions of the lockstep ring by logical index (0 = oldest): s, a [n, 2], r, s2, d."""
        idx = np.ascontiguousarray(logical_idx, np.int64)
        n, o = idx.size, self.cfg.obs_dim
        s = np.zeros((n, o), np.float32); s2 = np.zeros((n, o), np.float32)
        a = np.zeros((n, 2), np.float32); r = np.zeros(n, np.float32); d = np.zeros(n, np.uint8)
        check(_lib.lib().uavrl_sac_replay_gather(self.h, n, _ptr(idx), _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d)))
        return s, a, r, s2, d

    def update_replay(self, idx_tape=None, eps_next=None, eps_cur=None, losses=None):
        """One update sampled from the lockstep ring (idx_tape: device int32 [batch_size] logical indices, or [G][batch_size]
        trainer-local ones; None = Philox)."""
        check(_lib.lib().uavrl_sac_update_replay(self.h, _ptr(idx_tape), _ptr(eps_next), _ptr(eps_cur), self._losses(losses),
                                                 _stream(self.device)))


def sac_smem_bytes(obs_dim, hidden, device=0):
    """Shared memory (dynamic + static bytes) one block of each SAC kernel takes for these networks: [target, critic update,
    actor update, get_action].  SacLearner refuses the shape when any exceeds 227 KB (232 448 B)."""
    c = _lib.SacConfig()
    c.obs_dim, c.hidden, c.act_dim, c.device = int(obs_dim), int(hidden), 2, int(device)
    out = np.zeros(4, np.int64)
    check(_lib.lib().uavrl_sac_smem_bytes(C.byref(c), _ptr(out)))
    return [int(x) for x in out]


def sac_train_run(env, sac, n_iters, do_update=True, want_stats=True):
    st = _lib.TrainStats()
    check(_lib.lib().uavrl_sac_train_run(env.h, sac.h, int(n_iters), int(bool(do_update)), C.byref(st) if want_stats else None,
                                         _stream(env.device)))
    return st
