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

    def set_reset_stride(self, stride):
        """Scenario advance of each env's auto-reset (default n).  A shard of N / W envs of an N-env batch, reset with
        first + r N / W, sets N and draws exactly the scenarios of its rows of the full batch."""
        check(_lib.lib().uavrl_env_set_reset_stride(self.h, int(stride)))

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

    # -- episode records (include/uavrl.h, uavrl_env_set_records): one per finished episode, written by the step
    def set_records(self, capacity):
        """capacity > 0: record every finished episode (episode j of env e in slot j n + e; slots >= capacity are dropped);
        0: off.  Enabling again empties them."""
        check(_lib.lib().uavrl_env_set_records(self.h, int(capacity)))
        self._rec_cap = int(capacity)

    def records(self, clear=True):
        """The written records in slot order as a dict of numpy columns (RECORD_FIELDS, plus 'slot'), with n_dropped; clear
        empties them and restarts the ordinals."""
        cap = getattr(self, "_rec_cap", 0)
        buf = (_lib.EpisodeRecord * max(cap, 1))()
        w, d = C.c_int64(), C.c_int64()
        check(_lib.lib().uavrl_env_get_records(self.h, cap, buf, C.byref(w), C.byref(d), int(bool(clear))))
        out = records_columns(buf, cap)
        out["n_dropped"] = int(d.value)
        return out

    def clear_records(self):
        check(_lib.lib().uavrl_env_clear_records(self.h))

    def threaten_rate(self, pts):
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        out = np.zeros(pts.shape[0], np.uint8)
        check(_lib.lib().uavrl_env_threaten_rate(self.h, pts.shape[0], _ptr(pts), _ptr(out)))
        return out

    # -- moving obstacles (include/uavrl.h, uavrl_env_set_motion): one table per batch, advanced once per step call
    def set_motion(self, velocity, positions=None):
        """velocity [n_buildings, 3]: every obstacle's `v` (motion on); None: motion off.  positions [n_buildings, 3] (z ignored):
        the centres to start from; None keeps the current ones.  Takes effect from the next step."""
        nb = self.city.buildings.shape[0]
        v = None if velocity is None else np.ascontiguousarray(velocity, np.float64).reshape(nb, 3)
        p = None if positions is None else np.ascontiguousarray(positions, np.float64).reshape(nb, 3)
        check(_lib.lib().uavrl_env_set_motion(self.h, _ptr(p), _ptr(v)))

    def obstacles(self):
        """(positions [n, 3] with z the base height, velocities [n, 3], step calls since set_motion) of the current table."""
        nb = self.city.buildings.shape[0]
        pos = np.zeros((nb, 3), np.float64); vel = np.zeros((nb, 3), np.float64)
        steps = C.c_int64()
        check(_lib.lib().uavrl_env_get_obstacles(self.h, _ptr(pos), _ptr(vel), C.byref(steps)))
        return pos, vel, int(steps.value)


RECORD_FIELDS = ("scenario", "env", "ordinal", "outcome", "steps", "subgoals", "collisions", "total_score", "path_len",
                 "start2goal", "planner_len", "final_dist", "energy")


def records_columns(buf, n, written_only=True):
    """numpy columns of the first n uavrl_episode_record entries of a ctypes array; 'slot' is each entry's index.
    written_only keeps the entries the step wrote (outcome != 0)."""
    arr = np.ctypeslib.as_array(buf)[:n] if n > 0 else np.zeros(0, dtype=np.ctypeslib.as_array(buf).dtype)
    keep = arr["outcome"] != 0 if written_only else np.ones(len(arr), bool)
    out = {k: np.array(arr[k][keep]) for k in RECORD_FIELDS}
    out["slot"] = np.nonzero(keep)[0].astype(np.int64)
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


class _PerCalls:
    """The prioritised-replay calls a learner handle shares with the other kind (SumTree + ReplayTree of the reference,
    BaseClass/replay_buffer.py:57-223): the C entry points named _PER + sample / set_errors / set_priorities / get, which take
    (n,) arrays on a one-trainer learner and (G, n) arrays of trainer-local slots on a learner with G > 1 trainers."""
    _PER = "uavrl_per_"

    def _per(self, name):
        return getattr(_lib.lib(), self._PER + name)

    def _per_shape(self, n):
        return (n,) if self.G == 1 else (self.G, n)

    def per_sample(self, batch, u_tape=None):
        """ReplayTree.sample2: (slots int32 [B], importance weights float32 [B]) on the device; (G, B) each on a grouped
        learner, u_tape (G, B)."""
        slots = torch.empty(self._per_shape(batch), dtype=torch.int32, device=self.device)
        w = torch.empty(self._per_shape(batch), dtype=torch.float32, device=self.device)
        check(self._per("sample")(self.h, int(batch), _ptr(u_tape), _ptr(slots), _ptr(w), _stream(self.device)))
        return slots, w

    def _per_n(self, slots):
        """Slots per trainer of a (n,) or, grouped, (G, n) slot array."""
        if self.G > 1 and (slots.dim() != 2 or slots.shape[0] != self.G):
            raise ValueError("a learner with %d trainers takes (%d, n) slots, got %s" % (self.G, self.G, tuple(slots.shape)))
        return int(slots.shape[-1])

    def per_set_errors(self, slots, abs_err, clip=True):
        check(self._per("set_errors")(self.h, self._per_n(slots), _ptr(slots), _ptr(abs_err), int(bool(clip)), _stream(self.device)))

    def per_set_priorities(self, slots, priorities):
        check(self._per("set_priorities")(self.h, self._per_n(slots), _ptr(slots), _ptr(priorities), _stream(self.device)))

    def per_state(self, n_slots):
        """(leaves, total, beta); grouped: n_slots per trainer, leaves (G, n_slots) and totals (G,)."""
        leaves = np.zeros(self._per_shape(int(n_slots)), np.float64)
        totals, beta = np.zeros(self.G, np.float64), C.c_double()
        check(self._per("get")(self.h, _ptr(leaves), totals.ctypes.data_as(C.POINTER(C.c_double)), C.byref(beta)))
        return leaves, (float(totals[0]) if self.G == 1 else totals), beta.value


class Learner(_PerCalls):
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
        probe_states, probe_tape = self._probe_sources(G, probe_states, probe_tape)
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

    def _probe_sources(self, G, probe_states, probe_tape):
        """Checked probe sources of an aggregation over G trainers: a host tape is checked and uploaded as int32."""
        if probe_tape is not None and not isinstance(probe_tape, torch.Tensor):
            tape = np.ascontiguousarray(probe_tape, np.int64)
            if tape.shape != (G, 10):
                raise ValueError("probe_tape must be (%d, 10), got %s" % (G, tape.shape))
            if any(len(set(row.tolist())) != 10 for row in tape):
                raise ValueError("probe_tape rows must hold 10 distinct indices")
            n_g = self.replay_size() // self.G
            if (tape < 0).any() or (tape >= n_g).any():
                raise ValueError("probe_tape indices must lie in [0, %d) (transitions per trainer)" % n_g)
            probe_tape = torch.from_numpy(tape.astype(np.int32)).to(self.device)
        if probe_states is not None and tuple(probe_states.shape) != (G, 10, self.in_dim):
            raise ValueError("probe_states must be (%d, 10, %d)" % (G, self.in_dim))
        return probe_states, probe_tape

    # -- the aggregation across trainers sharded over ranks (include/uavrl.h, uavrl_learner_fed_shard)
    def fed_shard(self, rank, world):
        """Declare this learner's trainers as the global trainers [rank G, (rank + 1) G) of G world (create it with
        seed + rank G).  Allocates, on the device and until the learner is closed or fed_shard runs again, the two exchange
        buffers of fed_exchange_tensor and the rounds' scratch: about 4 Gw^2 + 2 Gw (10 in_dim + 10 A + P) floats for
        Gw = G world trainers in all.  At Gw = 4096 and the 100-64-64-27 network that is 224 MB for exchange 0, 67 MB for
        exchange 1, and about 0.6 GB in all."""
        check(_lib.lib().uavrl_learner_fed_shard(self.h, int(rank), int(world)))
        self.fed_rank, self.fed_world = int(rank), int(world)

    def fed_exchange_tensor(self, phase):
        """The buffer all-gathered after fed_local (phase 0: [Gw, 10 in_dim + 10 A + P]) or fed_columns (phase 1:
        [world, Gw, G]), flat, as a torch view; this rank's slice is the rank-th of world equal parts."""
        n = C.c_int64()
        ptr = _lib.lib().uavrl_learner_fed_exchange_ptr(self.h, int(phase), C.byref(n))
        if not ptr:
            raise ValueError("fed_exchange_tensor needs fed_shard first and phase 0 or 1")
        return _DevView(ptr, n.value, self.device).tensor()

    def fed_local(self, probe_states=None, probe_tape=None, probe_idx=None):
        """Phase a: this rank's probe rows (probe_states (G, 10, in_dim), probe_tape (G, 10) device int32, or the ring),
        their Q and q_local into its slice of exchange 0.  probe_idx: optional (G, 10) int32 device output."""
        check(_lib.lib().uavrl_learner_fed_local(self.h, _ptr(probe_states), _ptr(probe_tape), _ptr(probe_idx), _stream(self.device)))

    def fed_columns(self):
        """Phase b, after the gather of exchange 0: this rank's columns of the initial losses into its slice of exchange 1."""
        check(_lib.lib().uavrl_learner_fed_columns(self.h, _stream(self.device)))

    def fed_rounds(self, losses=None, chosen=None):
        """Phase c, after the gather of exchange 1: every round, then this rank's q_local.  losses (Gw, Gw) float32 and chosen
        (Gw, max(1, k)) int32 device outputs may be None."""
        check(_lib.lib().uavrl_learner_fed_rounds(self.h, _ptr(losses), _ptr(chosen), _stream(self.device)))

    def federate_sharded(self, dist, probe_states=None, probe_tape=None, want_details=False):
        """federate() across the ranks of torch.distributed `dist` after fed_shard: every rank calls it, and every rank's
        trainers end where the one-GPU federate() of all Gw trainers leaves them, bit for bit.  probe_states (Gw, 10, in_dim)
        and probe_tape (Gw, 10) are global (each rank uses its own rows).  want_details: the global (probe_idx (Gw, 10),
        losses (Gw, Gw), chosen (Gw, max(1, k))) device tensors, as federate() returns them.  The rounds run on every rank,
        so the call costs what the one-GPU rounds cost, plus two all-gathers."""
        r, W, G = self.fed_rank, self.fed_world, self.G
        Gw = G * W
        probe_states, probe_tape = self._probe_sources(Gw, probe_states, probe_tape)
        mine = slice(r * G, (r + 1) * G)
        own = lambda t: None if t is None else t[mine].contiguous()  # noqa: E731
        idx = losses = chosen = None
        if want_details:
            idx = torch.empty((Gw, 10), dtype=torch.int32, device=self.device)
            losses = torch.empty((Gw, Gw), dtype=torch.float32, device=self.device)
            chosen = torch.empty((Gw, max(1, (Gw - 1) // 2)), dtype=torch.int32, device=self.device)
        self.fed_local(own(probe_states), own(probe_tape), None if idx is None else idx[mine])
        for phase in (0, 1):
            x = self.fed_exchange_tensor(phase)
            dist.all_gather_into_tensor(x, x.chunk(W)[r].clone())
            if phase == 0:
                self.fed_columns()
        self.fed_rounds(losses, chosen)
        if want_details:
            dist.all_gather_into_tensor(idx, idx[mine].clone())
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

    def per_enable_trainers(self, alpha=-1.0, beta0=-1.0, beta_inc=-1.0, eps=-1.0, err_upper=-1.0):
        """Prioritised replay with one tree per trainer (include/uavrl.h uavrl_per_enable_trainers); per_enable when G = 1.
        With G > 1 the per_* methods then take and return (G, ...) arrays of trainer-local slots."""
        check(_lib.lib().uavrl_per_enable_trainers(self.h, alpha, beta0, beta_inc, eps, err_upper))

    def compute_grads(self, global_batch, idx_tape=None, loss=None):
        check(_lib.lib().uavrl_learner_compute_grads(self.h, _ptr(idx_tape), int(global_batch), _ptr(loss),
                                                     _stream(self.device)))

    def grad_tensor(self):
        """The device gradient vector as a torch view (for torch.distributed.all_reduce)."""
        ptr = _lib.lib().uavrl_learner_grad_ptr(self.h)
        arr = (C.c_float * self.P).from_address(ptr) if False else None  # noqa: F841 (device memory: no host view)
        return _DevView(ptr, self.P, self.device).tensor()

    def _comm(self):
        lib = _lib.lib()
        return (64, lambda rank, world, h: lib.uavrl_learner_comm_init(self.h, rank, world, h, None),
                lambda handles: lib.uavrl_learner_comm_connect(self.h, handles, None))

    def connect_peers(self, dist, rank, world):
        """Exchange the CUDA IPC handles of the symmetric gradient receive buffers over torch.distributed and map
        every peer's buffer (NVLink P2P) -- enables update_dp(), the fused one-shot all-reduce + Adam."""
        _connect_peers(dist, rank, world, self.device, *self._comm())

    def connect_self(self):
        """world = 1: the data-parallel optimiser kernel (push into the local receive buffer, gather, all-reduce + Adam) on
        one GPU -- the self-test of the fused path that needs no second device."""
        _connect_peers(None, 0, 1, self.device, *self._comm())

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


def _connect_peers(dist, rank, world, device, nbytes, init, connect):
    """The handle exchange of the fused data-parallel optimiser, shared by Learner and SacLearner: init(rank, world, buf)
    writes this rank's nbytes-byte record (the CUDA IPC handle of its receive buffer, ...), every rank's record is gathered
    over torch.distributed in rank order, connect(records) maps every peer's buffer.  dist = None: world 1, no peers."""
    mine = (C.c_ubyte * nbytes)()
    check(init(rank, world, mine))
    if dist is None:
        check(connect(mine))
        return
    t = torch.tensor(list(bytes(mine)), dtype=torch.uint8, device=device)
    allh = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(allh, t)
    g = np.ascontiguousarray(torch.stack(allh).cpu().numpy())
    check(connect(_ptr(g)))
    dist.barrier(device_ids=[device.index])


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


class SacLearner(_PerCalls):
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

    # -- the actor aggregation across trainers sharded over ranks (include/uavrl.h, uavrl_sac_fed_shard)
    def fed_shard(self, rank, world):
        """Declare this learner's trainers as the global trainers [rank G, (rank + 1) G) of G world (create it with
        seed + rank G); allocates the exchange buffer of every global trainer's actor (G world Pa floats)."""
        check(_lib.lib().uavrl_sac_fed_shard(self.h, int(rank), int(world)))
        self.fed_rank, self.fed_world = int(rank), int(world)

    def fed_exchange_tensor(self):
        """The [G world, Pa] actor buffer, flat, as a torch view; this rank's slice is the rank-th of world equal parts."""
        n = C.c_int64()
        ptr = _lib.lib().uavrl_sac_fed_exchange_ptr(self.h, C.byref(n))
        if not ptr:
            raise ValueError("fed_exchange_tensor needs fed_shard first")
        return _DevView(ptr, n.value, self.device).tensor()

    def fed_local(self):
        """This rank's actors into its slice of the exchange buffer."""
        check(_lib.lib().uavrl_sac_fed_local(self.h, _stream(self.device)))

    def fed_sum_actors(self):
        """After the gather: every own actor becomes the sum of all G world actors in trainer order."""
        check(_lib.lib().uavrl_sac_federate_actors_sharded(self.h, _stream(self.device)))

    def federate_actors_sharded(self, dist):
        """federate_actors() across the ranks of torch.distributed `dist` after fed_shard: every rank's actors end as the
        one-GPU call on all trainers leaves them, bit for bit."""
        self.fed_local()
        x = self.fed_exchange_tensor()
        dist.all_gather_into_tensor(x, x.chunk(self.fed_world)[self.fed_rank].clone())
        self.fed_sum_actors()

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

    def act(self, obs, eps=None, mean=False):
        """SAC_Trainer.get_action on n rows; mean=True: the mean action tanh(mu) bound instead (act_mean)."""
        if mean:
            return self.act_mean(obs)
        n = obs.shape[0]
        a = torch.empty((n, self.cfg.act_dim), dtype=torch.float32, device=self.device)
        check(_lib.lib().uavrl_sac_act(self.h, _ptr(obs), n, _ptr(eps), _ptr(a), _stream(self.device)))
        return a

    def act_mean(self, obs):
        """The policy's mean action tanh(mu) bound (include/uavrl.h uavrl_sac_act_mean): no noise, no act-call counted."""
        a = torch.empty((obs.shape[0], self.cfg.act_dim), dtype=torch.float32, device=self.device)
        check(_lib.lib().uavrl_sac_act_mean(self.h, _ptr(obs), obs.shape[0], _ptr(a), _stream(self.device)))
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
        trainer-local ones; None = Philox, or the trees once per_enable has run)."""
        check(_lib.lib().uavrl_sac_update_replay(self.h, _ptr(idx_tape), _ptr(eps_next), _ptr(eps_cur), self._losses(losses),
                                                 _stream(self.device)))

    # -- prioritised replay (include/uavrl.h, uavrl_sac_per_enable): one SumTree per trainer over its slots of the ring
    _PER = "uavrl_sac_per_"

    def per_enable(self, alpha=-1.0, beta0=-1.0, beta_inc=-1.0, eps=-1.0, err_upper=-1.0):
        """Every update that samples the ring then draws from the trees, weights the critic losses and writes
        e_b = mean_j |min(Q1, Q2)_j - y_j| back; the per_* methods take (G, ...) arrays when G > 1."""
        check(_lib.lib().uavrl_sac_per_enable(self.h, alpha, beta0, beta_inc, eps, err_upper))

    def tree_slots(self):
        """Leaves of each trainer's tree: its slots of the ring, ring_frames x lockstep_envs / G (ReplayStore::alloc)."""
        Ng = self.cfg.lockstep_envs // self.G
        return (max(2, -(-(self.cfg.replay_capacity // self.G) // Ng)) + 1) * Ng

    def update_batch_per(self, s, a, r, s2, d, is_weights, abs_err_out=None, eps_next=None, eps_cur=None, losses=None):
        """update_batch with importance weights is_weights [B] in the critic losses and each row's e_b written to abs_err_out
        [B] (may be None); the trees are not touched."""
        check(_lib.lib().uavrl_sac_update_batch_per(self.h, s.shape[0], _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d), _ptr(is_weights),
                                                    _ptr(abs_err_out), _ptr(eps_next), _ptr(eps_cur), self._losses(losses),
                                                    _stream(self.device)))

    # -- data-parallel training (include/uavrl.h, uavrl_sac_comm_init .. uavrl_sac_train_run_dp): one learner per GPU
    def _comm(self):
        lib = _lib.lib()
        return (_lib.SAC_COMM_HANDLE_BYTES, lambda rank, world, h: lib.uavrl_sac_comm_init(self.h, rank, world, h),
                lambda handles: lib.uavrl_sac_comm_connect(self.h, handles))

    def connect_peers(self, dist, rank, world):
        """Exchange every rank's receive-buffer handle and device over torch.distributed and map the peers' buffers: enables
        update_replay_dp() and sac_train_run_dp(), two fused all-reduce + Adam exchanges per update.  Every rank needs its own
        GPU (refused otherwise)."""
        _connect_peers(dist, rank, world, self.device, *self._comm())

    def connect_self(self):
        """world = 1: the fused data-parallel update on one GPU (each exchange pushes into and gathers from the local buffer)."""
        _connect_peers(None, 0, 1, self.device, *self._comm())

    def update_replay_dp(self, global_batch, idx_tape=None, eps_next=None, eps_cur=None, losses=None):
        """One data-parallel update from this rank's ring: losses averaged over global_batch rows, gradients and loss sums
        summed over the ranks by the fused exchanges."""
        check(_lib.lib().uavrl_sac_update_replay_dp(self.h, _ptr(idx_tape), _ptr(eps_next), _ptr(eps_cur), int(global_batch),
                                                    self._losses(losses), _stream(self.device)))

    def critic_grads(self, global_batch, batch=None, idx_tape=None, eps_next=None):
        """Split form, phase 1: epoch += 1, then the critics' gradients and squared-error sums on batch = (s, a, r, s2, d)
        device tensors (kept alive until actor_grads) or, with batch None, on rows sampled from the ring; they land in
        exchange_tensor(0), which the caller sums over the ranks before apply_critic_grads()."""
        st = _stream(self.device)
        if batch is None:
            check(_lib.lib().uavrl_sac_critic_grads_replay(self.h, _ptr(idx_tape), _ptr(eps_next), int(global_batch), st))
        else:
            s, a, r, s2, d = batch
            check(_lib.lib().uavrl_sac_critic_grads_batch(self.h, s.shape[0], _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d),
                                                          _ptr(eps_next), int(global_batch), st))

    def apply_critic_grads(self):
        check(_lib.lib().uavrl_sac_apply_critic_grads(self.h, _stream(self.device)))

    def actor_grads(self, eps_cur=None):
        """Split form, phase 3: the actor leg on the same rows with the stepped critics, into exchange_tensor(1)."""
        check(_lib.lib().uavrl_sac_actor_grads(self.h, _ptr(eps_cur), _stream(self.device)))

    def apply_actor_grads(self, losses=None):
        """Split form, phase 4: the actor's Adam step, the alpha step, the soft target update and the global losses."""
        check(_lib.lib().uavrl_sac_apply_actor_grads(self.h, self._losses(losses), _stream(self.device)))

    def exchange_tensor(self, phase):
        """The device vector a phase exchanges, as a torch view: 0 = [grad critic_1 | grad critic_2 | their squared-error
        sums] (2 Pc + 2 floats), 1 = [grad actor | actor-loss sum, entropy sum] (Pa + 2)."""
        n = C.c_int64()
        ptr = _lib.lib().uavrl_sac_exchange_ptr(self.h, int(phase), C.byref(n))
        if not ptr:
            raise ValueError("phase must be 0 (critics) or 1 (actor)")
        return _DevView(ptr, n.value, self.device).tensor()


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


def sac_train_run_dp(env, sac, n_iters, global_batch):
    """uavrl_sac_train_run_dp: lockstep iterations whose update is the fused data-parallel SAC update (after connect_peers
    or connect_self; warm the ring up with sac_train_run first)."""
    check(_lib.lib().uavrl_sac_train_run_dp(env.h, sac.h, int(n_iters), int(global_batch), _stream(env.device)))


def _eval_result(env, learner, n_episodes, buf, st):
    """records in suite order (all n_episodes positions, unfinished ones with outcome 0), the trainer of each row and the stats"""
    out = records_columns(buf, n_episodes, written_only=False)
    del out["slot"]
    out["trainer"] = out["env"] // (env.n // learner.G)
    out["trainer"][out["outcome"] == 0] = -1
    return dict(records=out, iterations=int(st.iterations), n_records=int(st.records), unfinished=int(st.unfinished))


def eval_run(env, learner, n_episodes, first_scenario=0, max_iters=0):
    """uavrl_eval_run: greedy episodes of a Q-network learner over pool scenarios first_scenario + k (mod P), k < n_episodes,
    one record each.  Returns dict(records = numpy columns in suite order plus 'trainer' (-1: unfinished), iterations,
    n_records, unfinished).  Nothing of the learner changes; the env ends in the evaluation's final state."""
    n = int(n_episodes)
    buf = (_lib.EpisodeRecord * max(n, 1))()
    st = _lib.EvalStats()
    check(_lib.lib().uavrl_eval_run(env.h, learner.h, int(first_scenario), n, int(max_iters), buf, C.byref(st), _stream(env.device)))
    return _eval_result(env, learner, n, buf, st)


def sac_eval_run(env, sac, n_episodes, first_scenario=0, max_iters=0, mean_action=False):
    """uavrl_sac_eval_run: eval_run for a SAC learner; sampled actions on the evaluation's own noise stream, or with
    mean_action the mean action tanh(mu) bound."""
    n = int(n_episodes)
    buf = (_lib.EpisodeRecord * max(n, 1))()
    st = _lib.EvalStats()
    check(_lib.lib().uavrl_sac_eval_run(env.h, sac.h, int(first_scenario), n, int(bool(mean_action)), int(max_iters), buf, C.byref(st),
                                        _stream(env.device)))
    return _eval_result(env, sac, n, buf, st)
