"""Env plug-in: the reference's PathPlan_City (Envs/PathPlan_City.py) with `num_UAV` UAV instances
stepped in lockstep on a H100.  <num_trainers> (default 1) independent Q-network trainers share them: trainer g learns
from UAVs [g num_UAV / num_trainers, (g + 1) num_UAV / num_trainers) and is named UAV_<g num_UAV / num_trainers>.
num_trainers = num_UAV is the reference's one trainer per UAV (PathPlan_City.py:59-69); 1 is one shared trainer.

Constructor takes the same parsed-XML dict the reference's EnvFactory passes
(config/PathPlan_City.xml <env> ... </env>): len/width/h, num_UAV, Agent.xml_path_agent,
Agent.Trainer.Trainer_path, Obstacles.buildings.  simulator.py drives it unchanged:
env.run_eposide(eps) -> result dict; env.Agents[i].Train_time / Testing_time; env.Trainer.hard_update().
"""
import importlib
import math
import os
import time

import numpy as np
import torch

import uavrl_b200  # noqa: F401  (repository root must be on sys.path)
from uavrl_b200 import engine
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
        agents_params = param.get('Agent')
        self.uav_dict = XML2Dict(os.path.normpath(agents_params['xml_path_agent'])).get('Agent')
        self.uav_params = uav_params_from_dict(self.uav_dict)
        self.sub_granularity = int(None2Value(self.uav_dict.get("sub_granularity"), 30))
        fn = self.uav_dict.get("update_function_name")
        self.discrete = (fn != "update_PathPlan")            # update_PathPlan27: the discrete-27 extension
        self.batch = engine.EnvBatch(self.city, self.uav_params, self.num_UAV, max_subgoals=64,
                                     device=self.device_index, auto_reset=True)
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
        if power is not None or self.record_csv:
            self.batch.set_extras(power=power, track_envs=(1 if self.record_csv else 0),
                                  track_capacity=(64 * self.uav_params.max_step if self.record_csv else 0))
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
        tdict['n_trainers'] = str(self.num_trainers)
        tdict['lockstep_envs'] = '0' if self.host_driven else str(self.num_UAV)
        tdict['device'] = str(self.device_index)
        ttype = tdict.get('Trainer_Type')
        try:
            mod = importlib.import_module("uavrl_b200.plugins." + ttype)
        except ImportError:
            mod = importlib.import_module(ttype)
        self.Trainer = getattr(mod, ttype)(tdict)
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
        self.executed_time = 0
        self.Scene_Random_Reset()

    # ---- geometry the planners use
    def Threaten_rate(self, p):
        return int(self.batch.threaten_rate([[p.x, p.y, p.z]])[0])

    # ---- reset / observation / step for all UAVs
    def Scene_Random_Reset(self):
        """UAV.reset() for the whole batch (a new block of the scenario pool).  Individual UAVs whose
        episode ends restart by themselves inside the step kernel."""
        self.batch.reset(self._next_first)
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
        if is_sac == self.discrete:
            raise ValueError("SAC needs update_function_name = update_PathPlan (continuous); the DQN family needs update_PathPlan27")
        if self.host_driven:
            raise ValueError("run_eposide drives the device-resident lockstep loop: construct without host_driven")
        t0 = time.time()
        save_loop = int(getattr(self.Trainer, "save_loop", 0) or 0)
        ended = steps = updates = coll = n_s = n_l = 0
        reward_sum, loss, chunk, iters = 0.0, 0.0, 16, 0
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
            ended += st.episodes_ended; steps += st.env_steps; updates += st.updates; coll += st.collisions
            n_s += st.n_success; n_l += st.n_lose; reward_sum += st.sum_reward; loss = st.last_loss
            iters += chunk
        dt = time.time() - t0
        ag = self.Agents[0]
        ag.Train_time += dt
        ag.score = reward_sum / max(1, ended)
        ag.Step = iters
        self.result.update(success=n_s, lose=n_l, normal=steps - n_s - n_l, loss=float(loss),
                           sum_epoch=self.Trainer.epoch, score=reward_sum, average_score=reward_sum / self.num_UAV,
                           step=iters, env_steps=steps, updates=updates, collisions=coll, episodes=ended)
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

    def Federated_Learning_choice(self):
        """PathPlan_City.py:644-684 on the device (engine.Learner.federate): every trainer averages itself with the half of
        the other trainers whose Q-values lie closest to its own on 10 states of its replay.  The reference's run_eposide calls
        Federated_Learning (:475), which cannot run (sample2 unpacking, trainer methods the reference lacks); this plug-in runs
        the reference's selective aggregation instead.  One trainer (or the SAC trainer) has nothing to aggregate with."""
        learner = self.Trainer._learner
        if isinstance(learner, engine.SacLearner) or learner.trainer_count() < 2:
            return
        learner.federate()

    def Federated_Learning_AC(self):
        """PathPlan_City.py:590-601 on the device (engine.SacLearner.federate_actors): every SAC trainer's actor is replaced by
        the sum of all trainers' actors.  The reference divides by the trainer count into a temporary state_dict, so the
        division is lost and the sum is what it trains on; this plug-in reproduces that.  Critics, targets, Adam moments and
        alpha are untouched; one trainer keeps its actor."""
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
