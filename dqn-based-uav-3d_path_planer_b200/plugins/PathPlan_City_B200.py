"""Env plug-in: the reference's PathPlan_City (Envs/PathPlan_City.py) with `num_UAV` UAV instances
stepped in lockstep on a H100.  <num_trainers> (default 1) independent Q-network trainers share them: trainer g learns
from UAVs [g num_UAV / num_trainers, (g + 1) num_UAV / num_trainers) and is named UAV_<g num_UAV / num_trainers>.
num_trainers = num_UAV is the reference's one trainer per UAV (PathPlan_City.py:59-69); 1 is one shared trainer.
<shard_over_ranks>1</shard_over_ranks> spreads the UAVs and the trainers over the W ranks of an initialised torch.distributed
group (one process per GPU): rank r steps UAVs [r num_UAV / W, (r + 1) num_UAV / W) and trains trainers
[r num_trainers / W, (r + 1) num_trainers / W), each computing what the one-GPU run's trainer of that index computes.

Constructor takes the same parsed-XML dict the reference's EnvFactory passes
(config/PathPlan_City.xml <env> ... </env>): len/width/h, num_UAV, Agent.xml_path_agent,
Agent.Trainer.Trainer_path, Obstacles.buildings.  simulator.py drives it unchanged:
env.run_eposide(eps) -> result dict; env.Agents[i].Train_time / Testing_time; env.Trainer.hard_update().
env.run_evaluation(n) plays n held-out scenarios with the trained policy on an env of its own (<eval_seed>, <eval_episodes>,
<eval_envs>, <eval_mean_action>) and returns its summary; <record_episodes>1</record_episodes> adds generate_train_result's
per-episode fields to run_eposide's result.
Moving obstacles: a <Threaten> of the buildings XML may carry the `v` attribute UAV.cal_force reads, <v><x/><y/><z/></v>
(missing: zero).  <APF_Enabled>1</APF_Enabled> in the UAV XML turns the APF model on with those velocities, and
<moving_obstacles>1</moving_obstacles> in the env XML moves every obstacle by its `v` once per lockstep step (include/uavrl.h,
uavrl_env_set_motion).
"""
import importlib
import math
import os
import time

import numpy as np
import torch

import uavrl_b200  # noqa: F401  (repository root must be on sys.path)
from uavrl_b200 import engine
from uavrl_b200.plugins._trainer_base import TrainerB200
from uavrl_b200.plugins.xmlconfig import None2Value, XML2Dict


class UAVBatchView:
    """What simulator.py / PathPlan_City read from an Agent, aggregated over the batch."""

    def __init__(self, env, name="UAV_batch"):
        self.env, self.name = env, name
        self.Train_time = 0.0        # UAV.py:124-125, accumulated by run_eposide
        self.Testing_time = 0.0
        self.Trainer = env.Trainer
        self.score = 0.0
        self.Step = 0
        self.done = False
        self.UEs = []
        self.task_collect = 0
        self.transition_dict = {'states': [], 'actions': [], 'next_states': [], 'rewards': [], 'dones': []}

    @property
    def path(self):
        st = self.env.batch.get_state()
        return np.stack([st["px"], st["py"], st["pz"]], 1).tolist()

    def state(self):
        return self.env.states()

    @property
    def energy_cost_total(self):
        """UAV.energy_cost_total (Agents/UAV.py:93) summed over the batch: the accumulated Calc_Fly_Power (UAV.py:239-245) when
        the UAV XML carries <Power_param><Fly_power>, else 0 like the reference (which never accumulates it)."""
        return self.env.batch.get_energy_total() if self.env.energy_enabled else 0

    @energy_cost_total.setter
    def energy_cost_total(self, v):
        pass

    # UAV.Init_Record_Mod / record_list (Agents/UAV.py:269-307): logs/<name>_<time>.csv, one row per call
    CSV_HEADER = ["sum_Episode", "Episode", " Score", " Avg.Score", "eps-greedy", "success", "failed", "meet_threaten", 'loss', 'ALL_UEs_D',
                  'ALL_UEs_F', 'energy_cost', 'task_collect', 'Energy_Efficent', 'UE_waiting_time', 'Covered_rate', 'task_executed',
                  'executed_rate', 'KL', 'Train_time', 'Testing_time']

    def Init_Record_Mod(self, directory="logs"):
        import csv
        import datetime
        os.makedirs(directory, exist_ok=True)
        cur_time = datetime.datetime.now().strftime('%m_%d_%Y(%H_%M_%S)')
        self.csv_path = os.path.join(directory, '%s_%s.csv' % (self.name, cur_time))
        self._csv_file = open(self.csv_path, 'a+', newline="")
        self.CsvWriter = csv.writer(self._csv_file)
        self.CsvWriter.writerow(self.CSV_HEADER)

    def record_list(self):
        """One row in the reference's column order (UAV.py:280-307); the UE / task columns are 0 (no UEs on this path)."""
        if getattr(self, "CsvWriter", None) is None:
            return
        res = self.env.result
        energy = self.energy_cost_total
        self.CsvWriter.writerow([self.Trainer.epoch, self.Trainer.epoch, self.score, self.score, res.get('eps', 0), res.get('success', 0),
                                 res.get('lose', 0), res.get('meet_threaten', 0), res.get('loss', 0), 0, 0, energy, self.task_collect,
                                 self.task_collect / (energy + 0.001), 0, 0, 0, 0, [], self.Train_time, self.Testing_time])
        self._csv_file.flush()

    def reset(self):
        self.env.Scene_Random_Reset()


def uav_params_from_dict(uav: dict):
    """Agents/UAV.py:25-32: Max_V int(), Steering_angle degrees -> rad, Max_Step int()."""
    return engine.UavParams(max_v=int(uav.get("Max_V")), min_v=float(None2Value(uav.get("Min_V"), 0.6)),
                            steering=float(uav.get("Steering_angle")) / 180 * math.pi,
                            climb_rate=float(None2Value(uav.get("climb_rate"), 1.0)), max_step=int(uav.get("Max_Step")))


def buildings_from_dict(bdict: dict):
    """Obstacles/building.py:8-11 for every <Threaten> of config/buildings.xml."""
    th = bdict["Threaten"]
    if isinstance(th, dict):
        th = [th]
    return np.array([[float(t["position"]["x"]), float(t["position"]["y"]), float(t["position"]["z"]),
                      float(None2Value(t.get("_R"), 10)), float(None2Value(t.get("_H"), 20))] for t in th], np.float64)


def obstacle_v_from_dict(bdict: dict):
    """The `v` of every <Threaten> ([n, 3], zero where it has none) and whether any of them has one."""
    th = bdict["Threaten"]
    if isinstance(th, dict):
        th = [th]
    vs = [t.get("v") for t in th]
    v = np.array([[float(None2Value(x.get(k), 0)) for k in ("x", "y", "z")] if isinstance(x, dict) else [0.0, 0.0, 0.0]
                  for x in vs], np.float64).reshape(-1, 3)
    return v, any(isinstance(x, dict) for x in vs)


def eval_summary(rec, num_trainers=1):
    """The summary run_evaluation returns, from evaluation records in suite order (engine.eval_run's 'records'): counts and
    rates over the finished episodes, means of their steps / path_len / total_score / start2goal / energy, the mean
    path_len / planner_len over successful episodes with a planner path, and with num_trainers > 1 each trainer's success
    rate."""
    done = rec["outcome"] != 0
    succ = rec["outcome"] == 1
    n = int(done.sum())

    def mean(x, m):
        return float(np.mean(x[m])) if m.any() else 0.0
    ratio_m = succ & (rec["planner_len"] > 0)
    out = dict(episodes=n, success=int(succ.sum()), lose=int((rec["outcome"] == 2).sum()), success_rate=float(succ.sum()) / max(n, 1),
               collisions=int(rec["collisions"][done].sum()), steps=mean(rec["steps"], done), path_len=mean(rec["path_len"], done),
               total_score=mean(rec["total_score"], done), start2goal=mean(rec["start2goal"], done),
               path_ratio=mean(rec["path_len"] / np.where(ratio_m, rec["planner_len"], 1.0), ratio_m), energy=mean(rec["energy"], done))
    if num_trainers > 1:
        out["success_rate_per_trainer"] = [float(succ[rec["trainer"] == g].sum()) / max(int(done[rec["trainer"] == g].sum()), 1)
                                           for g in range(num_trainers)]
    return out


def write_eval_csv(rec, path):
    """One row per finished episode: its suite position, then every record field and the trainer."""
    import csv
    cols = list(engine.RECORD_FIELDS) + ["trainer"]
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["position"] + cols)
        for k in np.nonzero(rec["outcome"] != 0)[0]:
            w.writerow([int(k)] + [rec[c][k].item() for c in cols])


class PathPlan_City_B200:
    def __init__(self, param: dict) -> None:
        # BaseEnv.__init__ (BaseClass/BaseEnv.py:19-21,34)
        self.len = int(None2Value(param.get("len"), 100))
        self.width = int(None2Value(param.get("width"), 100))
        self.h = int(None2Value(param.get("h"), 20))
        self.Is_AC = int(None2Value(param.get("Is_AC"), 0))
        self.eps = float(None2Value(param.get('eps'), 0.1))
        self.Is_On_Policy = int(None2Value(param.get('Is_On_Policy'), 0))
        if self.Is_On_Policy:
            raise ValueError("PathPlan_City_B200 implements the off-policy (DQN-family) loop only")
        self.param = param
        self.device_index = int(None2Value(param.get("device"), 0))
        # buildings (PathPlan_City.py:43-51)
        bpath = os.path.normpath(param['Obstacles']['buildings'])
        self.buildings_param = XML2Dict(bpath).get('buildings')
        self.buildings_table = buildings_from_dict(self.buildings_param)
        self.city = engine.City(self.len, self.width, self.h, self.buildings_table)
        # agents (PathPlan_City.py:54-69)
        self.num_UAV = int(param.get('num_UAV'))
        self.num_trainers = int(None2Value(param.get('num_trainers'), 1))
        if self.num_trainers < 1 or self.num_UAV % self.num_trainers != 0:
            raise ValueError("num_UAV (%d) must be a multiple of num_trainers (%d)" % (self.num_UAV, self.num_trainers))
        # shard_over_ranks = 1: this rank's share of the UAVs and trainers.  Its env shard draws the scenarios of its rows of the
        # whole batch (reset stride num_UAV), its trainers are seeded and named by their global index, the episode loop sums
        # its counts over the ranks once per chunk, and the aggregations run across the ranks (federate_sharded)
        self.shard_over_ranks = int(None2Value(param.get('shard_over_ranks'), 0))
        self.rank, self.world, self._dist = 0, 1, None
        if self.shard_over_ranks:
            import torch.distributed as dist
            if not (dist.is_available() and dist.is_initialized()):
                raise ValueError("shard_over_ranks = 1 needs an initialised torch.distributed process group")
            self.rank, self.world, self._dist = dist.get_rank(), dist.get_world_size(), dist
            if self.num_UAV % self.world or self.num_trainers % self.world:
                raise ValueError("shard_over_ranks = 1 needs num_UAV (%d) and num_trainers (%d) to be multiples of the world size "
                                 "(%d)" % (self.num_UAV, self.num_trainers, self.world))
            if param.get("device") is None:
                self.device_index = torch.cuda.current_device()
        self.n_local = self.num_UAV // self.world              # the UAVs this process steps
        agents_params = param.get('Agent')
        self.uav_dict = XML2Dict(os.path.normpath(agents_params['xml_path_agent'])).get('Agent')
        self.uav_params = uav_params_from_dict(self.uav_dict)
        # APF_Enabled (UAV.py:448-453) with the obstacles' `v`; moving_obstacles = 1: the obstacles move by it every step
        self.obstacle_v, has_v = obstacle_v_from_dict(self.buildings_param)
        self.apf_enabled = int(None2Value(self.uav_dict.get("APF_Enabled"), 0))
        self.moving_obstacles = int(None2Value(param.get("moving_obstacles"), 0))
        if self.apf_enabled and not has_v:
            raise ValueError("APF_Enabled = 1 needs obstacle velocities: no <Threaten> of the buildings XML carries a <v>")
        self.sub_granularity = int(None2Value(self.uav_dict.get("sub_granularity"), 30))
        fn = self.uav_dict.get("update_function_name")
        self.discrete = (fn != "update_PathPlan")            # update_PathPlan27: the discrete-27 extension
        self.batch = engine.EnvBatch(self.city, self.uav_params, self.n_local, max_subgoals=64,
                                     device=self.device_index, auto_reset=True)
        if self.shard_over_ranks:
            self.batch.set_reset_stride(self.num_UAV)
        self.pool_size = int(None2Value(param.get("scenario_pool"), max(1024, 2 * self.num_UAV)))
        sc = self.batch.make_scenarios(self.pool_size, seed=int(None2Value(param.get("seed"), 42)),
                                       rrt_step=self.sub_granularity)
        self.batch.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
        self._next_first = 0
        # optional models of the UAV (uavrl_env_set_extras): the energy model when the UAV XML carries the reference's
        # <Power_param><Fly_power> block (config/UAV.xml:27-36), trajectory recording for path.csv when record_csv = 1
        self.record_csv = int(None2Value(param.get("record_csv"), 0))
        fp = (self.uav_dict.get("Power_param") or {}).get("Fly_power") if isinstance(self.uav_dict.get("Power_param"), dict) else None
        self.energy_enabled = fp is not None
        power = None
        if fp is not None:
            power = {k: float(fp[k]) for k in ("P_i", "v_0", "d_0", "rho", "s", "A", "P_b", "F_b")}
            power["xi"] = 0.8                                      # UAV.py:58 with j = 0 (one shared parameter set)
        self._power = power
        self._apf_v = self.obstacle_v if self.apf_enabled else None
        if power is not None or self.record_csv or self.apf_enabled:
            self.batch.set_extras(power=power, obstacle_v=self._apf_v, track_envs=(1 if self.record_csv else 0),
                                  track_capacity=(64 * self.uav_params.max_step if self.record_csv else 0))
        if self.moving_obstacles:
            self.batch.set_motion(self.obstacle_v)
        # trainer(s): one handle holding num_trainers independent trainers
        tpath = os.path.normpath(agents_params['Trainer']['Trainer_path'])
        tdict = XML2Dict(tpath).get('Trainer')
        tdict['name'] = 'UAV_0'
        # host_driven = 1: the per-step methods (states / Move_Agents / Trainer.get_action / replay_memory.add / update) carry
        # HOST arrays across every boundary like the reference's own objects, and the trainer keeps the generic replay store;
        # 0 (default): run_eposide drives the device-resident lockstep loop (observations go straight into the replay ring)
        self.host_driven = int(None2Value(param.get('host_driven'), 0))
        if self.host_driven and self.num_trainers > 1:
            raise ValueError("host_driven = 1 drives one trainer: it needs num_trainers = 1")
        if self.host_driven and self.shard_over_ranks:
            raise ValueError("host_driven = 1 drives one process's host arrays: it cannot shard over ranks (set shard_over_ranks = 0)")
        g_local = self.num_trainers // self.world
        tdict['n_trainers'] = str(g_local)
        tdict['lockstep_envs'] = '0' if self.host_driven else str(self.n_local)
        if self.shard_over_ranks:
            tdict['first_trainer'] = str(self.rank * g_local)
            tdict['seed'] = str(int(None2Value(tdict.get('seed'), 42)) + self.rank * g_local)
        tdict['device'] = str(self.device_index)
        ttype = tdict.get('Trainer_Type')
        try:
            mod = importlib.import_module("uavrl_b200.plugins." + ttype)
        except ImportError:
            mod = importlib.import_module(ttype)
        tcls = getattr(mod, ttype)
        if self.host_driven and not issubclass(tcls, TrainerB200):
            # run_step_OffPolicy needs the trainer's host replay facade and learn_off_policy, which only the DQN family has
            raise ValueError("host_driven = 1 drives the DQN-family trainers (DQN_Trainer_B200, DDQN_Trainer_B200, "
                             "DuelingDQN_Trainer_B200); %s has no host replay or learn_off_policy: set host_driven = 0" % ttype)
        self.Trainer = tcls(tdict)
        self.Agents = [UAVBatchView(self)]
        if self.record_csv:
            self.Agents[0].Init_Record_Mod()
        self.result = {}
        self.epoch = 0
        self.print_loop = int(None2Value(param.get('print_loop'), 2))
        # federated aggregation every FL_Loop episodes (PathPlan_City.py:78-79, :469-475).  With DQN-family trainers it runs the
        # reference's selective aggregation Federated_Learning_choice (:644-684) across the num_trainers trainers; with SAC
        # trainers and Is_AC = 1 the reference's Federated_Learning_AC (:590-601)
        self.Is_FL = int(None2Value(param.get('Is_FL'), 0))
        self.FL_Loop = int(None2Value(param.get('FL_Loop'), 3))
        if self.Is_FL:
            if self.FL_Loop < 1:
                raise ValueError("FL_Loop must be >= 1 when Is_FL = 1")
            if self.Is_AC and not isinstance(self.Trainer._learner, engine.SacLearner):
                raise ValueError("Is_FL = 1 with Is_AC = 1 averages the trainers' actors (Federated_Learning_AC), which DQN-family "
                                 "trainers do not have: set Is_AC = 0")
            if self.shard_over_ranks:
                self.Trainer._learner.fed_shard(self.rank, self.world)
        # evaluation (run_evaluation): a held-out pool drawn from eval_seed, eval_episodes suite episodes on eval_envs envs of
        # an env of its own; record_episodes = 1: run_eposide adds generate_train_result's per-episode fields
        seed = int(None2Value(param.get("seed"), 42))
        self.eval_seed = int(None2Value(param.get("eval_seed"), seed + 1))
        self.eval_episodes = int(None2Value(param.get("eval_episodes"), self.num_UAV))
        self.eval_envs = int(None2Value(param.get("eval_envs"), self.num_UAV))
        self.eval_mean_action = int(None2Value(param.get("eval_mean_action"), 0))
        self.record_episodes = int(None2Value(param.get("record_episodes"), 0))
        self._chunk = 16                                           # lockstep iterations per run_eposide chunk
        if self.eval_envs < 1 or self.eval_envs % self.num_trainers:
            raise ValueError("eval_envs (%d) must be a positive multiple of num_trainers (%d)" % (self.eval_envs, self.num_trainers))
        self._eval_batch = None
        if self.record_episodes:
            # a chunk ends at most `chunk` episodes per UAV, and run_eposide drains the records after every chunk: nothing drops
            self.batch.set_records(self._chunk * self.n_local)
        self.executed_time = 0
        self.Scene_Random_Reset()

    # ---- geometry the planners use
    def Threaten_rate(self, p):
        return int(self.batch.threaten_rate([[p.x, p.y, p.z]])[0])

    # ---- reset / observation / step for all UAVs
    def Scene_Random_Reset(self):
        """UAV.reset() for the whole batch (a new block of the scenario pool).  Individual UAVs whose
        episode ends restart by themselves inside the step kernel."""
        self.batch.reset(self._next_first + self.rank * self.n_local)
        self._next_first = (self._next_first + self.num_UAV) % self.pool_size
        self.Trainer._learner_reset_lockstep()

    def _host_out(self):
        """Pinned host staging for the step outputs, a ring of 4 sets (see TrainerB200._pinned): the arrays returned by
        states() / Move_Agents() are numpy views of these buffers and stay valid for the next 3 calls."""
        if not hasattr(self, "_hbuf"):
            N = self.num_UAV
            mk = lambda shape, dt: torch.empty(shape, dtype=dt, pin_memory=True)  # noqa: E731
            self._hbuf = [dict(obs=mk((N, engine.OBS_DIM), torch.float32), reward=mk((N,), torch.float32), done=mk((N,), torch.uint8),
                               info=mk((N,), torch.uint8)) for _ in range(4)]
            dev = self.batch.device
            self._dbuf = dict(obs=torch.empty((N, engine.OBS_DIM), dtype=torch.float32, device=dev),
                              reward=torch.empty(N, dtype=torch.float32, device=dev), done=torch.empty(N, dtype=torch.uint8, device=dev),
                              info=torch.empty(N, dtype=torch.uint8, device=dev))
            self._hturn = 0
        self._hturn = (self._hturn + 1) % 4
        return self._hbuf[self._hturn]

    def states(self):
        h = self._host_out()
        self.batch.observe(self._dbuf["obs"])
        h["obs"].copy_(self._dbuf["obs"], non_blocking=True)
        torch.cuda.current_stream(self.batch.device).synchronize()
        return h["obs"].numpy()

    def Move_Agents(self, actions, want_info_names=True):
        """BaseEnv.Move_Agent for every UAV: actions [N] (int32 indices or float32 steering) ->
        (next_states [N,100], rewards [N], dones [N], infos [N])."""
        a = np.asarray(actions)
        a = np.ascontiguousarray(a, np.int32 if self.discrete else np.float32)
        t = torch.from_numpy(a).to(self.batch.device, non_blocking=True)
        h = self._host_out()
        self.batch.step(t, out=self._dbuf)
        for k in ("obs", "reward", "done", "info"):
            h[k].copy_(self._dbuf[k], non_blocking=True)
        torch.cuda.current_stream(self.batch.device).synchronize()
        infos = h["info"].numpy()
        if want_info_names:
            infos = [engine.INFO_NAMES[i] for i in infos]
        return h["obs"].numpy(), h["reward"].numpy(), h["done"].numpy().view(np.bool_), infos

    # ---- one lockstep step with HOST arrays at every boundary (PathPlan_City.run_thread_OffPolicy :364-385 + update :757-776,
    #      for all UAVs at once): state -> Trainer.get_action -> Move_Agent -> replay add -> sample -> Trainer.update
    def run_step_OffPolicy(self, eps_rate, state=None):
        if not self.host_driven:
            raise ValueError("run_step_OffPolicy needs <host_driven>1</host_driven> (the lockstep ring belongs to run_eposide)")
        tr = self.Trainer
        s = self.states() if state is None else state                          # uav.state()
        a = tr.get_action(s, eps_rate)                                          # Choose_Action2 -> Trainer.get_action
        s2, r, d, info = self.Move_Agents(a, want_info_names=False)             # Move_Agent -> update + state
        tr.replay_memory.add_batch(s, a, r, s2, d)                              # replay_memory.add (:380-382)
        res = tr.learn_off_policy()                                             # sample + Trainer.update (:383-385, :757-776)
        return s2, r, d, info, res

    def Check_uav_Done(self):
        return bool(self.batch.get_state()["done"].all())

    def Reset_Result(self, eps_rate):
        self.result = {'success': 0, 'lose': 0, 'meet_threaten': 0, 'normal': 0, 'loss': 0, 'sum_epoch': 0,
                       'eps': eps_rate, 'score': 0, 'average_score': 0, 'step': 0}

    # ---- the episode loop (PathPlan_City.run_eposide :410-478, off-policy branch)
    def run_eposide(self, eps_rate=0.1):
        """One 'episode' of the batch: lockstep iterations (act -> step -> replay add -> update) until as
        many episodes ended as there are UAVs (every UAV finished one episode on average; finished UAVs
        restart from the scenario pool, which is the reference's per-episode UAV.reset())."""
        self.Reset_Result(eps_rate)
        learner = self.Trainer._learner
        is_sac = isinstance(learner, engine.SacLearner)
        if (is_sac and not learner.discrete) == self.discrete:
            raise ValueError("continuous SAC needs update_function_name = update_PathPlan (continuous); discrete SAC and the DQN "
                             "family need update_PathPlan27")
        if self.host_driven:
            raise ValueError("run_eposide drives the device-resident lockstep loop: construct without host_driven")
        t0 = time.time()
        save_loop = int(getattr(self.Trainer, "save_loop", 0) or 0)
        ended = steps = updates = coll = n_s = n_l = 0
        reward_sum, loss, chunk, iters = 0.0, 0.0, self._chunk, 0
        recs = []
        max_iters = 64 * self.uav_params.max_step
        while ended < self.num_UAV and iters < max_iters:
            e_before = self.Trainer.epoch
            if is_sac:
                st = engine.sac_train_run(self.batch, learner, chunk, bool(self.Trainer.Is_Train))
            else:
                # Is_Train = 0: get_action is greedy whatever eps is (uavrl_learner_set_is_train, set by the trainer plug-in)
                st = engine.train_run(self.batch, learner, chunk, eps_rate, 1, bool(self.Trainer.Is_Train))
            if not self.Trainer.Is_Train and not is_sac:
                # Trainer.update counts epochs whether or not it trains (DuelingDQN_Trainer.py:152)
                e, t = learner.counters()
                learner.set_counters(e_before + chunk, t)
            # the reference saves inside Trainer.update every save_loop epochs (DuelingDQN_Trainer.py:187-188, SAC_Trainer.py:436-437);
            # the device loop advances `chunk` epochs per call: save whenever a multiple of save_loop was crossed
            if save_loop > 0 and self.Trainer.epoch // save_loop != e_before // save_loop:
                self.Trainer.save()
            c = [st.episodes_ended, st.env_steps, st.collisions, st.n_success, st.n_lose, st.sum_reward, st.last_loss]
            if self._dist is not None:                             # every rank stops at the chunk the one-GPU run stops at
                t = torch.tensor(c, dtype=torch.float64, device=self.batch.device)
                self._dist.all_reduce(t)
                c = t.tolist()
                c[:5] = [int(x) for x in c[:5]]
                c[6] /= self.world                                 # the mean of the ranks' mean trainer losses
            if self.record_episodes:
                recs.append(self.batch.records(clear=True))
            ended += c[0]; steps += c[1]; updates += st.updates; coll += c[2]
            n_s += c[3]; n_l += c[4]; reward_sum += c[5]; loss = c[6]
            iters += chunk
        dt = time.time() - t0
        ag = self.Agents[0]
        ag.Train_time += dt
        ag.score = reward_sum / max(1, ended)
        ag.Step = iters
        self.result.update(success=n_s, lose=n_l, normal=steps - n_s - n_l, loss=float(loss),
                           sum_epoch=self.Trainer.epoch, score=reward_sum, average_score=reward_sum / self.num_UAV,
                           step=iters, env_steps=steps, updates=updates, collisions=coll, episodes=ended)
        if self.record_episodes:
            # generate_train_result (PathPlan_City.py:479-506): path_len, start2goal, len_Astar (the planner's polyline) and
            # ReachGoal, here the means over the episodes that ended in this call
            cat = {k: np.concatenate([r[k] for r in recs]) for k in ("path_len", "start2goal", "planner_len", "outcome")}
            m = (lambda x: float(np.mean(x)) if len(x) else 0.0)  # noqa: E731
            self.result.update(path_len=m(cat["path_len"]), start2goal=m(cat["start2goal"]), len_Astar=m(cat["planner_len"]),
                               ReachGoal=m(cat["outcome"] == 1))
        self.epoch += 1
        self.executed_time += dt
        if self.Is_FL and self.epoch % self.FL_Loop == 0:             # PathPlan_City.py:469-475
            if self.Is_AC and is_sac:
                self.Federated_Learning_AC()
            else:
                self.Federated_Learning_choice()
        if self.record_csv:
            self._write_path_csv()
            if self.print_loop > 0 and self.epoch % self.print_loop == 0:
                ag.record_list()                                   # PathPlan_City.run_eposide :463-468 (every print_loop episodes)
        return self.result

    # ---- policy evaluation: what the reference's Evaluation_Action / Sim stubs leave open
    def _eval_env(self):
        """The evaluation's own env, built once: the same city, UAV parameters and energy model, a pool from eval_seed."""
        if self._eval_batch is None:
            ev = engine.EnvBatch(self.city, self.uav_params, self.eval_envs, max_subgoals=64, device=self.device_index)
            sc = ev.make_scenarios(self.eval_episodes, seed=self.eval_seed, rrt_step=self.sub_granularity)
            ev.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
            if self._power is not None or self._apf_v is not None:
                ev.set_extras(power=self._power, obstacle_v=self._apf_v)
            self._eval_batch = ev
        return self._eval_batch

    def run_evaluation(self, n_episodes=None, log_dir="logs"):
        """The trained planner on n_episodes (default eval_episodes) held-out scenarios, each once, on the device: greedy for
        the DQN family, SAC's sampled action (eval_mean_action = 1: its mean action; discrete SAC: argmax p).  Neither the training env nor the
        trainer changes.  Returns eval_summary's dict plus the iterations run and the episodes left unfinished; writes one
        CSV row per episode to <log_dir>/eval_<time>.csv (CWD-relative, like the reference's logs) and adds the wall time
        to Agents[0].Testing_time."""
        if self.shard_over_ranks:
            raise ValueError("run_evaluation runs on one GPU: it is not available with shard_over_ranks = 1")
        if self.host_driven:
            raise ValueError("run_evaluation drives the device loop: it is not available with host_driven = 1")
        n = self.eval_episodes if n_episodes is None else int(n_episodes)
        if n > self.eval_episodes:
            raise ValueError("n_episodes (%d) exceeds the evaluation pool (eval_episodes = %d)" % (n, self.eval_episodes))
        t0 = time.time()
        ev, learner = self._eval_env(), self.Trainer._learner
        if self.moving_obstacles:                               # every evaluation starts from the XML table
            ev.set_motion(self.obstacle_v, positions=self.buildings_table[:, :3])
        if isinstance(learner, engine.SacLearner):
            res = engine.sac_eval_run(ev, learner, n, mean_action=bool(self.eval_mean_action))
        else:
            res = engine.eval_run(ev, learner, n)
        out = eval_summary(res["records"], self.num_trainers)
        out.update(iterations=res["iterations"], unfinished=res["unfinished"])
        path = os.path.join(log_dir, "eval_%s_%06d.csv" % (time.strftime("%Y%m%d-%H%M%S"), int(time.time() % 1 * 1e6)))
        write_eval_csv(res["records"], path)
        out["csv"] = path
        self.Agents[0].Testing_time += time.time() - t0
        return out

    def Federated_Learning_choice(self):
        """PathPlan_City.py:644-684 on the device (engine.Learner.federate): every trainer averages itself with the half of
        the other trainers whose Q-values lie closest to its own on 10 states of its replay.  The reference's run_eposide calls
        Federated_Learning (:475), which cannot run (sample2 unpacking, trainer methods the reference lacks); this plug-in runs
        the reference's selective aggregation instead.  One trainer (or the SAC trainer) has nothing to aggregate with."""
        learner = self.Trainer._learner
        if isinstance(learner, engine.SacLearner) or self.num_trainers < 2:
            return
        if self._dist is not None:
            learner.federate_sharded(self._dist)
        else:
            learner.federate()

    def Federated_Learning_AC(self):
        """PathPlan_City.py:590-601 on the device (engine.SacLearner.federate_actors): every SAC trainer's actor is replaced by
        the sum of all trainers' actors.  The reference divides by the trainer count into a temporary state_dict, so the
        division is lost and the sum is what it trains on; this plug-in reproduces that.  Critics, targets, Adam moments and
        alpha are untouched; one trainer keeps its actor."""
        if self._dist is not None:
            self.Trainer._learner.federate_actors_sharded(self._dist)
        else:
            self.Trainer._learner.federate_actors()

    def _write_path_csv(self, path="path.csv"):
        """UAV.py:461-464 / :479-482 / :505-508: at a terminal step the reference rewrites path.csv (CWD-relative) with the
        finished episode's UAV.path, one x,y,z row per step.  Here: the last finished episode of the tracked UAV 0."""
        import csv
        pts = self.batch.get_path(0, which=1)
        if len(pts) == 0:
            return
        with open(path, 'w', newline='') as f:
            w = csv.writer(f)
            for row in pts:
                w.writerow([float(row[0]), float(row[1]), float(row[2])])

    def run_XML_scene(self):
        pass

    def update(self):
        return [self.Trainer.learn_off_policy()]
