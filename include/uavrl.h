/* uavrl.h -- C ABI of the H100-native UAV path-planning hot path (libuavrl_b200.so).
 *
 * The reference (young-how/DQN-based-UAV-3D_path_planer, "RLGF") is pure Python with no FFI; its
 * hot path sits behind a duck-typed plug-in API resolved by name from XML (SURVEY.md section 8b).
 * This header is the boundary a reference-side plug-in binds with ctypes (INTEGRATION.md): plain
 * pointers and sizes only, no torch types.  Each entry point cites the reference interface it
 * replaces (paths relative to the reference repository root).
 *
 * Conventions
 *   - every function returns 0 on success or a negative uavrl_status; uavrl_last_error() gives the
 *     thread-local message.  Nothing falls back to a CPU path: without a CUDA device create() fails.
 *   - "_dev" pointers are device memory owned by the CALLER (e.g. torch.Tensor.data_ptr());
 *     "_host" pointers are host memory.  The library owns only its handles and their internal state.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  All work is
 *     enqueued on it; there are no hidden synchronisations except where a _host output is written.
 *   - one host thread per handle.
 *   - a call that runs out of device memory returns UAVRL_ERR_CUDA ("out of memory") and leaves the handle usable: a create
 *     frees everything it took, a call that replaces state (uavrl_env_set_pool, uavrl_env_generate_pool,
 *     uavrl_env_set_extras, uavrl_learner_comm_init, ...) leaves the old state in place, and scratch that failed to grow is
 *     grown again by the next call.
 */
#ifndef UAVRL_H
#define UAVRL_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UAVRL_OBS_DIM 100            /* Agents/UAV.py:517 state_map (1,1,1,100) */
#define UAVRL_MAX_HIDDEN 4

typedef enum {
    UAVRL_OK = 0,
    UAVRL_ERR_INVALID = -1,          /* bad argument / configuration */
    UAVRL_ERR_CUDA = -2,             /* CUDA runtime error (no device, launch failure, ...) */
    UAVRL_ERR_STATE = -3,            /* call order (e.g. step before reset) */
    UAVRL_ERR_NOMEM = -4
} uavrl_status;

typedef enum { UAVRL_INFO_NORMAL = 0, UAVRL_INFO_SUCCESS = 1, UAVRL_INFO_LOSE = 2 } uavrl_info;

/* action encodings accepted by uavrl_env_step */
typedef enum {
    UAVRL_ACT_CONT_F32 = 0,          /* steering fraction a0 = action[0] in [-1,1]  (UAV.py:407,414) */
    UAVRL_ACT_CONT_F64 = 1,          /* same, double (exact replay of reference tapes) */
    UAVRL_ACT_DISCRETE27 = 2,        /* int32 k in 0..26: documented extension, see DESIGN.md */
    UAVRL_ACT_CONT_F32X2 = 3         /* float [n][2] as SAC's get_action returns it; only action[0] steers (UAV.py:414) */
} uavrl_action_kind;

typedef enum { UAVRL_ALGO_DQN = 0, UAVRL_ALGO_DDQN = 1, UAVRL_ALGO_DUELING = 2 } uavrl_algo;

/* ------------------------------------------------------------------ environment batch */
typedef struct uavrl_env uavrl_env;

typedef struct {
    int32_t n_envs;                  /* UAV instances stepped in lockstep */
    int32_t max_subgoals;            /* K: capacity of each sub-goal queue (RRT path length bound) */
    double len, width, h;            /* BaseClass/BaseEnv.py:19-21 (config/PathPlan_City.xml:4-6) */
    double max_v, min_v;             /* config/UAV.xml:12-13 (Agents/UAV.py:25); 0 < max_v < 7 (the sub-goal radius: see uavrl_env_create) */
    double steering_angle;           /* radians: Steering_angle/180*pi (UAV.py:26) */
    int32_t max_step;                /* UAV.py:32 */
    double climb_rate;               /* discrete-27 extension only */
    int32_t n_buildings;
    const double *buildings_host;    /* [n][5] = cx, cy, cz, _R, _H (Obstacles/building.py:8-11) */
    int32_t device;                  /* CUDA device ordinal */
    int32_t auto_reset;              /* 1: an env whose episode ended (UAV.done) restarts from the
                                        scenario pool inside the same step call */
} uavrl_env_config;

int uavrl_env_create(const uavrl_env_config *cfg, uavrl_env **out);
int uavrl_env_destroy(uavrl_env *env);

/* Scenario pool = pre-generated outcomes of UAV.reset() (UAV.py:335-366): start ~U(10,210)x U(1,10),
 * goal ~U(330,490)x U(420,490), heading ~U(0,2pi), sub-goal queue from RRT (PathPlan/RRT.py:63-105;
 * queue[0] is the start point -- the very Loc object of the UAV, `alias0`=1 -- and the last entry
 * is the goal).  Host arrays: start[P][3], goal[P][3], heading[P], subgoals[P][K][3], n_sub[P],
 * alias0[P] (NULL = all 1). */
int uavrl_env_set_pool(uavrl_env *env, int32_t n_scenarios, const double *start_host,
                       const double *goal_host, const double *heading_host,
                       const double *subgoals_host, const int32_t *n_sub_host,
                       const uint8_t *alias0_host);

/* UAV.reset() for every env: env e takes scenario (first_scenario + e) mod P of the pool. */
int uavrl_env_reset(uavrl_env *env, int32_t first_scenario, void *stream);
/* The scenario an env takes at each auto-reset: its current scenario + stride (mod P).  The stride defaults to n_envs, which
 * keeps every env of the batch on its own scenarios.  A shard of a larger batch (rank r of W, n_envs = N / W, reset with
 * first_scenario + r N / W) sets stride N and then draws exactly the scenarios of its rows of the N-env batch.  Refused with
 * UAVRL_ERR_INVALID for stride < 1.  Takes effect from the next step. */
int uavrl_env_set_reset_stride(uavrl_env *env, int32_t stride);

/* Host-side scenario generator (reset draws + RRT) for synthetic pools: statistical restatement of
 * UAV.py:344-360 + RRT.py:26-105 with a counter-based RNG (the reference's Python MT19937 stream is
 * not reproduced).  Writes the arrays uavrl_env_set_pool takes. */
int uavrl_make_scenarios(const uavrl_env_config *cfg, uint64_t seed, int32_t n_scenarios,
                         int32_t rrt_step, double *start_host, double *goal_host,
                         double *heading_host, double *subgoals_host, int32_t *n_sub_host);

/* The same generator as a device kernel (one thread per scenario, SURVEY.md 8f-1): fills the env's device pool
 * directly -- replaces uavrl_make_scenarios + uavrl_env_set_pool, bit-identical scenarios for the same
 * (seed, index); replaces UAV.reset (UAV.py:335-366) + RRTPlanner.getPath (PathPlan/RRT.py:63-105) for the pool.
 * Synchronises `stream`.  uavrl_env_get_pool copies the current pool back (any pointer may be NULL):
 * start[P][3], goal[P][3], v0[P][3] = (Vx, Vy, |V|), subgoals[P][K][3], n_sub[P]. */
int uavrl_env_generate_pool(uavrl_env *env, int32_t n_scenarios, uint64_t seed, int32_t rrt_step, void *stream);
int uavrl_env_get_pool(uavrl_env *env, double *start_host, double *goal_host, double *v0_host,
                       double *subgoals_host, int32_t *n_sub_host);

/* UAV.state() -> state_PathPlan (UAV.py:515-567): obs_dev [n_envs][100] float32. */
int uavrl_env_observe(uavrl_env *env, float *obs_dev, void *stream);

/* BaseEnv.Move_Agent (BaseEnv.py:123-137) = UAV.update_PathPlan (UAV.py:397-513) followed by
 * UAV.state(), for all envs.  Outputs (any may be NULL): next_obs [n][100] f32, reward [n] f32,
 * done [n] u8 (the RETURNED flag, True at every sub-goal), info [n] u8 (uavrl_info),
 * collision [n] u8 (predicate at UAV.py:425), ended [n] u8 (UAV.done after the step, before any
 * auto-reset). */
int uavrl_env_step(uavrl_env *env, int32_t action_kind, const void *actions_dev,
                   float *next_obs_dev, float *reward_dev, uint8_t *done_dev, uint8_t *info_dev,
                   uint8_t *collision_dev, uint8_t *ended_dev, void *stream);

/* Same call with HOST buffers: copies actions in, runs the step, copies results out, synchronises.
 * This is the call a reference-side plug-in makes per lockstep iteration. */
int uavrl_env_step_host(uavrl_env *env, int32_t action_kind, const void *actions_host,
                        float *next_obs_host, float *reward_host, uint8_t *done_host,
                        uint8_t *info_host, uint8_t *collision_host, uint8_t *ended_host);

/* fp64 state read-back for parity tests / checkpoints; any pointer may be NULL.  Each [n_envs]. */
typedef struct {
    double *px, *py, *pz, *vx, *vy, *V, *score, *total_score, *path_len, *reward64;
    int32_t *step, *cursor, *scenario;
    uint8_t *done;
} uavrl_env_state_host;
int uavrl_env_get_state(uavrl_env *env, const uavrl_env_state_host *out);
/* Overwrite per-UAV state from host arrays (NULL members are left alone): position, V_vector / V, Step, score,
 * total_score, path_len, done -- the attributes UAV.reset / update_PathPlan maintain (Agents/UAV.py:335-366, 397-513);
 * resume from a saved state, or start a step from a constructed one.  The sub-goal queue, goal and cursor belong to the
 * scenario (uavrl_env_set_pool + uavrl_env_reset): cursor / scenario / reward64 must be NULL.  Synchronises the device. */
int uavrl_env_set_state(uavrl_env *env, const uavrl_env_state_host *in);

/* Optional models of the UAV (off by default; set after uavrl_env_create, before uavrl_env_reset):
 *   energy   UAV.Calc_Fly_Power (Agents/UAV.py:239-245) with the constants of config/UAV.xml <Power_param><Fly_power>
 *            (xi = 0.8 + 0.02 j, UAV.py:58): P(V) = P_i sqrt(sqrt(1 + V^4/(4 v_0^4)) - V^2/(2 v_0^2)) + d_0 rho s A V^3 / 2
 *            + xi P_b (1 + 3 V^2 / F_b^2), accumulated per step into a per-UAV energy column (the reference evaluates the
 *            formula but never accumulates it, UAV.py:59,93 -- the accumulator is the north-star's "energy model" output).
 *   apf      moving-obstacle artificial potential field (UAV.cal_force / Adjust_subgoal, UAV.py:156-210, and the reward
 *            term :448-453): obstacle_v_host [n_buildings][3] = the `v` attribute of each obstacle; obstacles with v = 0
 *            exert no force (UAV.py:180-182).  Every step shifts each remaining sub-goal by the force at its position,
 *            so sub-goal queues become per-UAV state.  The obstacles stay where they are unless uavrl_env_set_motion moves
 *            them; while it does, obstacle_v must equal its velocities.
 *   track    UAV.path (UAV.py:432) of the first track_envs UAVs, up to track_capacity points per episode, double
 *            buffered: the episode in progress and the last finished one (what path.csv holds, UAV.py:461-464). */
typedef struct {
    int32_t energy_enabled;
    double P_i, v_0, d_0, rho, s, A, P_b, F_b, xi;
    int32_t apf_enabled;
    const double *obstacle_v_host;
    int32_t track_envs, track_capacity;
} uavrl_env_extras;
int uavrl_env_set_extras(uavrl_env *env, const uavrl_env_extras *extras);
/* energy_host [n_envs]: sum of Calc_Fly_Power(V) over the steps of the episode in progress (joules per unit step time) */
int uavrl_env_get_energy(uavrl_env *env, double *energy_host);
/* flight energy of all UAVs over all steps since uavrl_env_create (the sum of UAV.energy_cost_total over the batch) */
int uavrl_env_get_energy_total(uavrl_env *env, double *total_out);
/* which = 0: episode in progress, 1: last finished episode.  xyz_host [capacity][3]; *n_out = points recorded */
int uavrl_env_get_path(uavrl_env *env, int32_t e, int32_t which, int32_t capacity, double *xyz_host, int32_t *n_out);
/* the per-UAV sub-goal queues [n_envs][K][3] (the scenario's queue, shifted by APF when enabled) */
int uavrl_env_get_subgoals(uavrl_env *env, double *sub_host);

/* Episode records: the per-episode statistics of the reference's UAV (Agents/UAV.py:147-153, 360-366, 443, 477, 503), which
 * PathPlan_City.generate_train_result (Envs/PathPlan_City.py:479-506) reads for Train_info_line.  With records on, the step
 * writes one record when an env's episode ends (UAV.done becomes true), before any auto-reset:
 *   scenario, env, ordinal   pool index, env row, and the env's ordinal-th finished episode since records were enabled or cleared
 *   outcome                  uavrl_info of the final step (1 success, 2 lose)
 *   steps                    step calls of the episode, over all its sub-goal segments (UAV.Step restarts at each sub-goal)
 *   subgoals                 sub-goals popped (the cursor's advance)
 *   collisions               steps whose collision predicate held (UAV.py:425)
 *   total_score, path_len    UAV.total_score and UAV.path_len at the end
 *   start2goal               Eu_Loc_distance(start, goal) of the scenario (UAV.start2goal, UAV.py:365)
 *   planner_len              calculate_path_len of the scenario's sub-goal queue, left to right (UAV.len_Astar, UAV.py:153,366:
 *                            the RRT sub-goal polyline, despite the name -- RRT.getPath returns the same list twice)
 *   final_dist               |p - goal| at the end
 *   energy                   the episode's Calc_Fly_Power sum with the energy model on, else 0
 * Episode j of env e goes to slot j n_envs + e; a record whose slot is at or beyond `capacity` is not written and counts as
 * dropped.  Slots are deterministic, so identical runs return identical arrays.  Records ride on the optional-model step (as
 * `track` does): with them off, the step is the default one.  They also work inside uavrl_train_run and uavrl_sac_train_run,
 * whose training outputs they do not change.
 * uavrl_env_set_records: capacity > 0 enables (or re-enables, emptied), capacity = 0 disables.  Synchronises the device.
 * uavrl_env_get_records: copies the min(capacity, slots) first slots to records_host (outcome 0: a slot not written), the
 * written and dropped counts, and with clear = 1 empties them (ordinals restart at 0).  uavrl_env_clear_records: the same
 * emptying alone.  Both synchronise the device; without records enabled they are refused (UAVRL_ERR_STATE). */
typedef struct {
    int32_t scenario, env, ordinal, outcome;
    int32_t steps, subgoals, collisions, reserved;
    double total_score, path_len, start2goal, planner_len, final_dist, energy;
} uavrl_episode_record;
int uavrl_env_set_records(uavrl_env *env, int64_t capacity);
int uavrl_env_get_records(uavrl_env *env, int64_t capacity, uavrl_episode_record *records_host, int64_t *n_written_out,
                          int64_t *n_dropped_out, int32_t clear);
int uavrl_env_clear_records(uavrl_env *env);

/* PathPlan_City.Threaten_rate (Envs/PathPlan_City.py:215-223) on arbitrary points (device kernel):
 * pts_host [n][3] -> out_host [n] u8. */
int uavrl_env_threaten_rate(uavrl_env *env, int32_t n, const double *pts_host, uint8_t *out_host);

/* Moving obstacles.  The reference's hooks for scene change (PathPlan_City.run(), BaseThreaten.run()) are `pass`; this is the
 * port's rule, built from the reference's own primitives.
 *   world    The n_envs UAVs of a batch are the UAVs of one city: one obstacle table per env handle.  It advances once per
 *            step call (uavrl_env_step, _step_host, the training and evaluation loops), whatever each env's episode is doing;
 *            uavrl_env_reset leaves it alone, and uavrl_env_observe / uavrl_env_threaten_rate read it without advancing it.
 *   state    Each obstacle has a centre (x, y) and a velocity (vx, vy, vz).  Its base z, _R and _H are fixed: cylinders stand on
 *            the ground (check_threaten tests p.z against the absolute _H), so vz moves nothing; it only adds to |v| in the APF.
 *   run()    Per obstacle, each IEEE operation rounded, in this order: x' = x + vx; if x' < 0 then x' = -x', vx = -vx; else if
 *            x' > len then x' = len - (x' - len), vx = -vx; then y likewise against width.  A reflection only flips signs, so
 *            |v| is constant; the APF direction of v, cos / sin of calculate_angle(0, v), is evaluated on the host with libm
 *            for all four sign variants (+-vx, +-vy) and the step selects one by the current signs.
 *   order    Within step t the UAV move, the collision test (UAV.py:425), the reward (APF term included) and Adjust_subgoal use
 *            the table O_t.  Every obstacle then runs once, giving O_{t+1}, and the observation the step writes (its probes,
 *            and the observation of an env that auto-resets in the step) uses O_{t+1}: it is s' of transition t and s of step
 *            t + 1.  With the table first set to the reference's positions after its first run(), the observation after k
 *            steps is the reference loop's state_test of iteration k.  (The reference's stored next_state is computed inside
 *            Move_Agent, before the next run(), against the old table; the port stores the observation the agent acts on.)
 * uavrl_env_set_motion: position_host [n_buildings][3] (z ignored) or NULL to keep the current centres; velocity_host
 *   [n_buildings][3] turns motion on, NULL turns it off (then position_host must be NULL too, and the step reads the cylinders
 *   as uavrl_env_create was given them).  Refused with UAVRL_ERR_INVALID, changing nothing: non-finite values, a centre
 *   outside [0, len] x [0, width], |vx| > len or |vy| > width, and velocities that differ from the APF model's obstacle_v
 *   while APF is on (uavrl_env_set_extras likewise refuses an obstacle_v that differs from these velocities while motion is
 *   on).  With both on, APF's force reads the moving table: current centres and current signs.  Motion rides on the
 *   optional-model step.  Synchronises the device; takes effect from the next step.
 * uavrl_env_get_obstacles: the current table, position_host [n][3] (z = the base height), velocity_host [n][3] (zero with
 *   motion off), and the step calls since uavrl_env_set_motion; any pointer may be NULL.  Synchronises the device. */
int uavrl_env_set_motion(uavrl_env *env, const double *position_host, const double *velocity_host);
int uavrl_env_get_obstacles(uavrl_env *env, double *position_host, double *velocity_host, int64_t *steps_out);

/* ------------------------------------------------------------------ learner (Q-net + replay) */
typedef struct uavrl_learner uavrl_learner;

typedef struct {
    int32_t in_dim;                       /* w (config/Trainer.xml <w>) */
    int32_t n_hidden;                     /* trunk layers with ReLU: Qnet2/VAnet2 = 1, QValueNet_SAC/VAnet3 = 2 ... */
    int32_t hidden[UAVRL_MAX_HIDDEN];     /* e.g. {64}, {64,64}, {128,64} (BaseClass/BaseCNN.py) */
    int32_t n_actions;                    /* <output> */
    int32_t dueling;                      /* 1: fc_A + fc_V heads, Q = V + A - mean(A) (BaseCNN.py:131-139) */
    int32_t algo;                         /* uavrl_algo */
    float lr;                             /* LEARNING_RATE (BaseTrainer.py:33) */
    float gamma;                          /* BaseTrainer.py:35 */
    int32_t batch_size;                   /* Batch_Size (BaseTrainer.py:34) */
    int32_t update_loop;                  /* hard target update period (DuelingDQN_Trainer.py:30,183) */
    int64_t replay_capacity;              /* replay_size, in transitions (BaseTrainer.py:32,39) */
    int32_t lockstep_envs;                /* >0: frame-ring replay fed by uavrl_train_* (N envs per frame);
                                             0: generic transition store fed by uavrl_replay_push */
    uint64_t seed;                        /* Philox key for eps-greedy and replay sampling */
    int32_t device;
    int32_t loss_kind;                    /* 0 = MSE, what every reference trainer uses (BaseTrainer.py:40, DQN_Trainer.py:119);
                                             1 = Huber / torch SmoothL1Loss(beta = 1): 0.5 d^2 for |d| < 1, |d| - 0.5 otherwise
                                             (an option the reference does not have; off for parity) */
} uavrl_learner_config;

int uavrl_learner_create(const uavrl_learner_config *cfg, uavrl_learner **out);
int uavrl_learner_destroy(uavrl_learner *l);
int64_t uavrl_learner_param_count(const uavrl_learner *l);

/* G independent trainers of the same network and hyper-parameters in one handle (PathPlan_City.py:59-69 builds one Trainer per
 * UAV; several seeds or replicas trained side by side).  uavrl_learner_create is n_trainers = 1.  The lockstep envs are split
 * into G contiguous blocks of Ng = lockstep_envs / G: trainer g acts for envs [g Ng, (g + 1) Ng), samples only their
 * transitions and owns its local and target parameters, Adam moments, gradient and loss.  epoch, adam_step and the
 * hard-update schedule are shared (the trainers step in lockstep).  Trainer g computes bit for bit what a stand-alone learner
 * with its parameters, seed + g, replay_capacity / G and Ng envs computes.  With G > 1:
 *   - set/get_params move [G][P] floats;
 *   - uavrl_learner_act takes n rows in G equal blocks (block g -> trainer g);
 *   - uavrl_learner_update_batch takes G B rows, block g for trainer g (B = rows / G);
 *   - uavrl_learner_update: idx_tape_dev is [G][batch_size] trainer-local logical indices; the k-th oldest transition of
 *     trainer g is the ring's logical index (k / Ng) N + g Ng + k % Ng (uavrl_replay_gather keeps whole-ring indices);
 *   - loss_dev receives [G] losses; uavrl_train_stats.last_loss is their mean;
 *   - replay_capacity is the total over trainers, and an update runs once every trainer holds more than batch_size
 *     transitions (replay size / G > batch_size);
 *   - uavrl_learner_tc_route describes one trainer's kernels for a per-trainer size n;
 *   - refused with UAVRL_ERR_INVALID: n_trainers outside [1, 65535] (one grid row per trainer), lockstep_envs % n_trainers != 0, uavrl_per_enable,
 *     uavrl_learner_update_batch_per, uavrl_replay_push, uavrl_learner_comm_init / comm_connect / update_dp / compute_grads /
 *     apply_grads, uavrl_train_run_dp, and act / update_batch sizes that are not multiples of G;
 *   - prioritised replay is enabled with uavrl_per_enable_trainers (one tree per trainer, trainer-local slots and [G][...] arrays
 *     in every uavrl_per_* call; see the prioritised-replay block).  uavrl_per_enable keeps refusing G > 1 because the grouped
 *     form changes the slot numbering and array shapes of the other uavrl_per_* calls, so a caller opts in by name. */
int uavrl_learner_create_trainers(const uavrl_learner_config *cfg, int32_t n_trainers, uavrl_learner **out);
int32_t uavrl_learner_trainer_count(const uavrl_learner *l);

/* Selective federated aggregation across the G trainers (Envs/PathPlan_City.py:644-684, Federated_Learning_choice; Is_FL with
 * a DQN-family trainer).  Rounds p = 0, 1, ..., G-1, in this order and in place:
 *   - probes: 10 distinct transitions of trainer p's own replay (random.sample(memory, 10)), their state rows;
 *   - q_value = Q(theta_p, probes) with theta_p as it stands (it changes only in round p);
 *   - loss_q = mean((q_value - Q(theta_q, probes))^2) over 10 x A for every q != p, theta_q trainer q's CURRENT q_local:
 *     for q < p the parameters round q already replaced;
 *   - the trainers sorted by (loss, index) -- Python's stable sort keeps equal losses in ascending q -- and the first
 *     k = (G - 1) / 2 kept;
 *   - theta_p <- (theta_p + theta_c0 + theta_c1 + ...) / (k + 1), per element a float32 left-to-right sum in the sorted
 *     order and one float32 division (bit-reproducible).
 * Only q_local and its kernel-layout images change (replace_param, :683; the reference's averaged q_target is discarded):
 * q_target, the Adam moments, epoch and adam_step are untouched.  G = 1 returns 0 and does nothing; G = 2 has k = 0 and
 * leaves every parameter as it is.
 *   probe_states_dev   [G][10][in_dim] explicit probe states (block p for round p), or NULL: draw them from the lockstep ring;
 *   probe_tape_dev     ring mode only, or NULL: [G][10] trainer-local logical indices (the convention of
 *                      uavrl_learner_update's tape: in range [0, replay size / G) and distinct within a row -- not checked on
 *                      the device).  NULL: Philox draws keyed by seed + g and a per-learner federation call counter;
 *   probe_idx_out_dev  optional [G][10]: the trainer-local indices used (-1 with explicit probe states);
 *   loss_out_dev       optional [G][G]: row p = the losses round p ranked, [p][p] = 0;
 *   chosen_out_dev     optional [G][max(1, k)]: round p's chosen trainers in sorted order (-1 when k = 0).
 * Everything is enqueued on `stream` (about 5 G kernel launches; the cost grows as G^2), with no host synchronisation.
 * Refused with UAVRL_ERR_INVALID before anything is enqueued: both probe sources given; ring mode on a learner without a
 * lockstep ring or with fewer than 10 transitions per trainer. */
int uavrl_learner_federate(uavrl_learner *l, const float *probe_states_dev, const int32_t *probe_tape_dev,
                           int32_t *probe_idx_out_dev, float *loss_out_dev, int32_t *chosen_out_dev, void *stream);

/* The same aggregation over trainers spread across ranks (one trainer group per UAV group, the groups sharded over GPUs).
 * Rank r's learner of G_local trainers holds the global trainers [r G_local, (r + 1) G_local) of G = G_local world: create it
 * with seed + r G_local.  uavrl_learner_fed_shard declares the shard once and allocates the buffers below (freed with the
 * handle, replaced by a later call); refused with UAVRL_ERR_INVALID for world < 1, rank outside [0, world) or G > 65535.
 * One aggregation is three calls with two all-gathers between them, which the caller makes in rank order into the buffers
 * uavrl_learner_fed_exchange_ptr returns (phase 0 or 1; NULL before uavrl_learner_fed_shard; len_out = floats in all, rank r's
 * slice is the r-th of world equal parts):
 *   uavrl_learner_fed_local     probe states of the own trainers (from the ring as uavrl_learner_federate draws them, or the
 *                               own rows [G_local][10][in_dim] / [G_local][10] of explicit states or a tape; probe_idx_out
 *                               [G_local][10] as there), their Q, and q_local: [probes | q_ref | q_local] per trainer into
 *                               exchange 0 = [G][10 in_dim + 10 A + P] (13 649 floats per trainer at 100-64-64-27);
 *   uavrl_learner_fed_columns   after the gather of exchange 0: the initial losses of the own trainers' columns into exchange
 *                               1 = [world][G][G_local];
 *   uavrl_learner_fed_rounds    after the gather of exchange 1: rounds p = 0 .. G-1, run redundantly on every rank, then the
 *                               own q_local and images.  loss_out [G][G] and chosen_out [G][max(1, k)] as uavrl_learner_federate.
 * Every rank ends with the parameters, losses and chosen lists the one-GPU call on all G trainers produces, bit for bit.
 * Device memory per rank: about 4 G^2 + 2 G (10 in_dim + 10 A + P) floats.  Refused with UAVRL_ERR_STATE before
 * uavrl_learner_fed_shard or out of order (columns need local, rounds need columns; local may restart at any time), and
 * with UAVRL_ERR_INVALID as uavrl_learner_federate refuses its probe sources; a refused call changes nothing. */
int uavrl_learner_fed_shard(uavrl_learner *l, int32_t rank, int32_t world);
float *uavrl_learner_fed_exchange_ptr(uavrl_learner *l, int32_t phase, int64_t *len_out);
int uavrl_learner_fed_local(uavrl_learner *l, const float *probe_states_dev, const int32_t *probe_tape_dev,
                            int32_t *probe_idx_out_dev, void *stream);
int uavrl_learner_fed_columns(uavrl_learner *l, void *stream);
int uavrl_learner_fed_rounds(uavrl_learner *l, float *loss_out_dev, int32_t *chosen_out_dev, void *stream);

/* state_dict()-ordered flat fp32 parameters (fc1.weight [out][in], fc1.bias, ..., for dueling nets
 * ..., fc_A.weight, fc_A.bias, fc_V.weight, fc_V.bias) -- what torch.save({'model': ...}) holds
 * (DuelingDQN_Trainer.py:79-84).  which: 0 = q_local, 1 = q_target, 2 = Adam exp_avg,
 * 3 = Adam exp_avg_sq, 4 = last gradient. */
int uavrl_learner_set_params(uavrl_learner *l, int32_t which, const float *params_host);
int uavrl_learner_get_params(uavrl_learner *l, int32_t which, float *params_host);
int uavrl_learner_set_counters(uavrl_learner *l, int64_t epoch, int64_t adam_step);
int uavrl_learner_get_counters(uavrl_learner *l, int64_t *epoch, int64_t *adam_step);

/* Trainer.get_action (DuelingDQN_Trainer.py:86-97) for n observations: u > eps (or !is_train)
 * -> argmax_a q_local(obs), else a uniformly random action.  u_tape_dev / rand_tape_dev inject the
 * random draws (parity tests); NULL = Philox.  q_out_dev optional [n][A]. */
int uavrl_learner_act(uavrl_learner *l, const float *obs_dev, int32_t n, float eps, int32_t is_train,
                      const float *u_tape_dev, const int32_t *rand_tape_dev, int32_t *actions_dev,
                      float *q_out_dev, void *stream);

/* ReplayMemory.add (BaseClass/replay_buffer.py:41-42), n transitions, FIFO over replay_capacity. */
int uavrl_replay_push(uavrl_learner *l, int32_t n, const float *obs_dev, const int32_t *actions_dev,
                      const float *reward_dev, const float *next_obs_dev, const uint8_t *done_dev,
                      void *stream);
int64_t uavrl_replay_size(const uavrl_learner *l);
/* Read back n stored transitions by logical index (0 = oldest) into host arrays (checkpointing the
 * replay, tests): s/s2 [n][in], a [n], r [n], d [n]. */
int uavrl_replay_gather(uavrl_learner *l, int32_t n, const int64_t *logical_idx_host, float *s_host,
                        int32_t *a_host, float *r_host, float *s2_host, uint8_t *d_host);

/* Trainer.update (DuelingDQN_Trainer.py:150-190; DQN_Trainer.py:85-136; DDQN_Trainer.py:72-117):
 * epoch += 1; sample Batch_Size distinct transitions uniformly (replay_buffer.py:48-51;
 * idx_tape_dev injects the indices, NULL = Philox), TD target, MSE loss, backward, Adam step, hard
 * target update every update_loop epochs.  Skipped (epoch still counts) while the replay holds
 * <= Batch_Size transitions (PathPlan_City.py:383).  loss_dev optional [1]. */
int uavrl_learner_update(uavrl_learner *l, const int32_t *idx_tape_dev, float *loss_dev, void *stream);

/* The same update on an explicit batch (transition_dict of DuelingDQN_Trainer.update): device arrays
 * s [B][in], a [B], r [B], s2 [B][in], d [B] (float 0/1). */
int uavrl_learner_update_batch(uavrl_learner *l, int32_t B, const float *s_dev, const int32_t *a_dev,
                               const float *r_dev, const float *s2_dev, const float *d_dev,
                               float *loss_dev, void *stream);

/* Split form for data-parallel training: grads only (sum over the local batch of d(loss)/d(theta),
 * loss normalised by global_batch), then -- after the caller all-reduced uavrl_learner_grad_ptr()
 * across ranks -- the optimiser step.  Unlike uavrl_learner_update, compute_grads refuses a replay holding
 * <= batch_size transitions with UAVRL_ERR_STATE, before the epoch counts: every rank must take part in every
 * exchange, and a rank that retries keeps the other ranks' sample keys and target-update schedule. */
int uavrl_learner_compute_grads(uavrl_learner *l, const int32_t *idx_tape_dev, int32_t global_batch,
                                float *loss_dev, void *stream);
float *uavrl_learner_grad_ptr(uavrl_learner *l);          /* device, [param_count] fp32 */
int uavrl_learner_apply_grads(uavrl_learner *l, void *stream);
/* Select the arithmetic path of the Q-network forward passes (get_action, TD target): 1 = wgmma tensor
 * cores with the 3xTF32 split (default when the network fits), 0 = fp32 CUDA cores.  Returns the path in use. */
int uavrl_learner_set_tensor_cores(uavrl_learner *l, int32_t enable);
int uavrl_learner_hard_update(uavrl_learner *l, void *stream);   /* DuelingDQN_Trainer.py:199-202 */
/* Trainer.Is_Train (BaseTrainer.py:47) for the lockstep loops below: with 0, get_action is greedy whatever eps is
 * (`sample > eps or not self.Is_Train`, DuelingDQN_Trainer.py:90).  Default 1. */
int uavrl_learner_set_is_train(uavrl_learner *l, int32_t is_train);
/* After an explicit uavrl_env_reset the lockstep ring's current frame no longer matches the env
 * state: call this; the next uavrl_train_run re-observes into a fresh frame and the lockstep replay
 * restarts empty (envs that end episodes restart by themselves with auto_reset and need no call). */
int uavrl_learner_lockstep_restart(uavrl_learner *l);

/* One-shot NVLink all-reduce fused with the optimiser (data-parallel training, one process per GPU):
 *   uavrl_learner_comm_init     allocate this rank's symmetric receive buffer recv[2][world][P+1] of 8-byte words, return its
 *                               CUDA IPC handle (64 bytes) for exchange (e.g. torch.distributed.all_gather)
 *   uavrl_learner_comm_connect  open every rank's handle (grad_handles: [world][64] bytes)
 *   uavrl_learner_update_dp     epoch += 1; local gradient (loss scaled by 1/global_batch), then ONE optimiser kernel: each
 *                               block reduces its slice of the gradient and PUSHES it with remote stores over NVLink into
 *                               slot `rank` of every rank's receive buffer, every value as one word {exchange tag : value};
 *                               it then polls its own receive buffer (local memory) until all `world` words of each of its
 *                               parameters carry the current tag, sums them in rank order (bit-identical replicas) and
 *                               applies Adam.  No NCCL call, no flag, no fence, nothing pulled across NVLink on the
 *                               critical path.  world = 1 runs the same kernel on the local buffer (self-test on one GPU).
 * flag_handle_out / flag_handles are unused (kept for ABI compatibility) and may be NULL.
 * loss_dev (optional) receives the GLOBAL batch loss.  update_dp refuses, before the epoch counts: a learner not connected
 * (UAVRL_ERR_STATE) and a replay holding <= batch_size transitions (UAVRL_ERR_STATE), as compute_grads does. */
int uavrl_learner_comm_init(uavrl_learner *l, int32_t rank, int32_t world, void *grad_handle_out, void *flag_handle_out);
int uavrl_learner_comm_connect(uavrl_learner *l, const void *grad_handles, const void *flag_handles);
int uavrl_learner_update_dp(uavrl_learner *l, const int32_t *idx_tape_dev, int32_t global_batch, float *loss_dev, void *stream);

/* ------------------------------------------------------------------ fused lockstep training loop
 * PathPlan_City.run_thread_OffPolicy + update (Envs/PathPlan_City.py:364-385,757-776) for all envs:
 *   obs -> get_action -> Move_Agent -> replay add -> [sample -> Trainer.update]
 * n_iters lockstep iterations; observations are written once, straight into the replay frame ring.
 * updates_per_iter optimiser steps follow each env step (reference: 1).  stats_host (optional)
 * receives the counters below. */
typedef struct {
    int64_t env_steps, updates, episodes_ended, collisions;
    int64_t n_success, n_lose;       /* steps whose info was 'success' / 'lose' (PathPlan_City.Run_statistics) */
    double sum_reward;
    float last_loss;
} uavrl_train_stats;
int uavrl_train_run(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps,
                    int32_t updates_per_iter, int32_t do_update, uavrl_train_stats *stats_host,
                    void *stream);

/* ------------------------------------------------------------------ SAC, continuous actions (BASELINE config 5)
 * SAC_Trainer (Trainer/SAC_Trainer.py) with PolicyNetContinuous_SAC / QValueNetContinuous_SAC (BaseClass/BaseCNN.py:459-500):
 * actor obs->hidden->{mu, sigma}, twin critics [obs, action]->hidden->hidden->action_dim, their targets, learnable log_alpha
 * (init ln 0.01).  The reference's quirks are kept: [B, action_dim]-shaped critic outputs / TD target / losses and the
 * doubly applied tanh in the log-prob correction. */
typedef struct uavrl_sac uavrl_sac;
typedef struct {
    int32_t obs_dim, hidden, act_dim;     /* <w>, <hiden_dim>, <output>/<action_dim> of config/Trainer.xml: 100, 64, 2 */
    float action_bound;                   /* <action_bound> */
    float actor_lr, critic_lr, alpha_lr;  /* actor.lr, critic.lr, SAC_param.alpha_lr */
    float target_entropy, gamma, tau;     /* SAC_param */
    int32_t batch_size;                   /* Batch_Size */
    int64_t replay_capacity;              /* replay_size */
    int32_t lockstep_envs;                /* > 0: frame-ring replay fed by uavrl_sac_train_run */
    uint64_t seed;
    int32_t device;
    int32_t discrete;                     /* 0: continuous actions (IS_Continuous = 1); 1: discrete actions (IS_Continuous = 0) */
} uavrl_sac_config;

/* Limits: obs_dim a multiple of 4 in [4, 124] (the critic input obs_dim + 2 is at most 128), hidden in [1, 128], and every
 * SAC kernel's shared memory (the networks are resident in it) at most 227 KB per block.  Refused with UAVRL_ERR_INVALID before
 * anything is allocated. */
int uavrl_sac_create(const uavrl_sac_config *cfg, uavrl_sac **out);
int uavrl_sac_destroy(uavrl_sac *s);
/* G independent SAC trainers of the same networks and hyper-parameters in one handle (PathPlan_City.py:59-69 builds one
 * SAC_Trainer per UAV).  uavrl_sac_create is n_trainers = 1.  The lockstep envs are split into G contiguous blocks of
 * Ng = lockstep_envs / G: trainer g acts for envs [g Ng, (g + 1) Ng), samples only their transitions and owns its actor, both
 * critics and both targets, their Adam moments and last gradients, its log_alpha with that scalar's Adam moments, and its
 * losses.  epoch and adam_step are shared (the trainers step in lockstep).  Trainer g computes bit for bit what a stand-alone
 * learner with its parameters and alpha, seed + g, replay_capacity / G and Ng envs computes.  With G > 1:
 *   - uavrl_sac_set/get_params move [G][P] floats for every role;
 *   - uavrl_sac_set/get_alpha move the [G][3] array {log_alpha, exp_avg, exp_avg_sq} (any G);
 *   - uavrl_sac_get_scalars reports trainer 0's alpha triple, uavrl_sac_set_scalars writes its triple to every trainer;
 *   - uavrl_sac_act takes n rows in G equal blocks (block g -> trainer g; eps_dev likewise);
 *   - uavrl_sac_update_batch takes G B rows, block g for trainer g (B = rows / G; eps_next / eps_cur likewise);
 *   - uavrl_sac_update_replay: idx_tape_dev is [G][batch_size] trainer-local logical indices; the k-th oldest transition of
 *     trainer g is the ring's logical index (k / Ng) N + g Ng + k % Ng (uavrl_sac_replay_gather keeps whole-ring indices);
 *   - losses_dev receives [G][4] losses; uavrl_train_stats.last_loss is the mean of the G actor losses;
 *   - replay_capacity is the total over trainers, and an update runs once every trainer holds more than batch_size
 *     transitions (replay size / G > batch_size);
 *   - refused with UAVRL_ERR_INVALID before anything is allocated: n_trainers outside [1, 65535] (one grid row per trainer),
 *     lockstep_envs % n_trainers != 0, replay_capacity / n_trainers == 0; and act / update_batch sizes that are not multiples
 *     of G. */
int uavrl_sac_create_trainers(const uavrl_sac_config *cfg, int32_t n_trainers, uavrl_sac **out);
int32_t uavrl_sac_trainer_count(const uavrl_sac *s);
/* Federated_Learning_AC (Envs/PathPlan_City.py:590-601; Is_FL = 1 with Is_AC = 1 and SAC trainers) across the G trainers.
 * The reference copies actor 0, adds actors 1 .. G-1 into the copy, and its division by G assigns into a temporary state_dict,
 * so nothing is divided: every trainer's actor becomes the float32 sum theta_0 + theta_1 + ... + theta_{G-1}, added left to
 * right in trainer order (bit-reproducible).  G = 1 leaves the actor as it is.  Critics, targets, every Adam moment, alpha,
 * epoch and adam_step are untouched.  Enqueued on `stream` (two launches), with no host synchronisation. */
int uavrl_sac_federate_actors(uavrl_sac *s, void *stream);
/* Federated_Learning_AC over trainers spread across ranks: rank r's learner of G_local trainers holds the global trainers
 * [r G_local, (r + 1) G_local) of G = G_local world (created with seed + r G_local).  uavrl_sac_fed_shard declares the shard and
 * allocates the exchange [G][Pa] (6 724 floats per trainer at the shipped shape; refused with UAVRL_ERR_INVALID for world < 1,
 * rank outside [0, world) or G > 65535); uavrl_sac_fed_exchange_ptr returns it (NULL before the shard; rank r's slice is the
 * r-th of world parts).  uavrl_sac_fed_local copies the own actors into the own slice; after the caller's all-gather,
 * uavrl_sac_federate_actors_sharded sums the G actors in trainer order 0 .. G-1, as uavrl_sac_federate_actors does, into every
 * own actor and its image.  Refused with UAVRL_ERR_STATE before the shard, or the sum without a local call since the last. */
int uavrl_sac_fed_shard(uavrl_sac *s, int32_t rank, int32_t world);
float *uavrl_sac_fed_exchange_ptr(uavrl_sac *s, int64_t *len_out);
int uavrl_sac_fed_local(uavrl_sac *s, void *stream);
int uavrl_sac_federate_actors_sharded(uavrl_sac *s, void *stream);
/* Shared memory (dynamic + static bytes) one block of each SAC kernel would take for cfg's networks: bytes_out[4] = target,
 * critic update, actor update, get_action.  uavrl_sac_create refuses cfg when any exceeds 227 KB (232 448 B). */
int uavrl_sac_smem_bytes(const uavrl_sac_config *cfg, int64_t *bytes_out);
/* role: 0 actor, 1 critic_1, 2 critic_2, 3 target_critic_1, 4 target_critic_2 (flat state_dict order:
 * actor = fc1, fc_mu, fc_std; critic = fc1, fc2, fc_out); 5..7 Adam exp_avg of actor/critic_1/critic_2, 8..10 exp_avg_sq;
 * 11..13 the gradients of actor/critic_1/critic_2 the last update reduced over its batch and fed to Adam (get only) */
int64_t uavrl_sac_param_count(const uavrl_sac *s, int32_t role);
int uavrl_sac_set_params(uavrl_sac *s, int32_t role, const float *params_host);
int uavrl_sac_get_params(uavrl_sac *s, int32_t role, float *params_host);
int uavrl_sac_set_scalars(uavrl_sac *s, float log_alpha, float la_exp_avg, float la_exp_avg_sq, int64_t epoch, int64_t adam_step);
int uavrl_sac_get_scalars(uavrl_sac *s, float *log_alpha, float *la_exp_avg, float *la_exp_avg_sq, int64_t *epoch, int64_t *adam_step);
/* every trainer's {log_alpha, Adam exp_avg, Adam exp_avg_sq}: [G][3] floats */
int uavrl_sac_set_alpha(uavrl_sac *s, const float *alpha_host);
int uavrl_sac_get_alpha(uavrl_sac *s, float *alpha_host);
/* SAC_Trainer.get_action (:444-448): actions_dev [n][2] = tanh(mu + sigma*eps)*bound; eps_dev [n][2] injects the
 * reparameterisation noise (NULL = Philox Box-Muller) */
int uavrl_sac_act(uavrl_sac *s, const float *obs_dev, int32_t n, const float *eps_dev, float *actions_dev, void *stream);

/* ------------------------------------------------------------------ SAC, discrete actions (discrete = 1)
 * SAC_Trainer with <IS_Continuous>0</IS_Continuous> (Trainer/SAC_Trainer.py:380-430, calc_target :133-141, get_action
 * :449-454) and PolicyNet_SAC / QValueNet_SAC (BaseClass/BaseCNN.py:296-343):
 *   actor   fc1 -> ReLU -> fc2 -> ReLU -> fc3 -> softmax over A       (obs -> hidden -> hidden -> A)
 *   critic  fc1 -> ReLU -> fc2 -> ReLU -> fc3, the A Q-values of s      (no action input), two of them and two targets
 * log_alpha starts at ln 0.01 with its own Adam (alpha_lr); there is no actor target.  One update on B rows (s, a in [0, A),
 * r, s', d), every float computed in fp32:
 *   1. reward shaping, a reference quirk kept (:390): r~ = (r + 10) / 10, inside the update only -- the ring, the env
 *      statistics and the episode records keep raw rewards;
 *   2. target: p' = actor(s'), H' = -sum_j p'_j log(p'_j + 1e-8) (the +1e-8 inside the log is the reference's),
 *      m' = sum_j p'_j min(Q1t(s'), Q2t(s'))_j, y = r~ + gamma (m' + alpha H') (1 - d), alpha = exp(log_alpha) before this
 *      update's alpha step;
 *   3. critics: L_k = mean_b (Q_k(s)[a_b] - y_b)^2; each critic takes its own Adam step -- BEFORE the actor's leg (kept);
 *   4. actor, on the UPDATED critics: p = actor(s), H and m as in 2 on s, L_pi = mean(-alpha H - m); gradients flow through p
 *      only: dL/dp_j = (alpha (log(p_j + 1e-8) + p_j / (p_j + 1e-8)) - min_j) / B, then the softmax Jacobian;
 *   5. alpha: L_alpha = mean((H - target_entropy) alpha), the gradient taken with respect to log_alpha, Adam on log_alpha;
 *   6. both targets move by tau toward the updated critics.
 * losses_dev receives {actor loss, critic 1 loss, critic 2 loss, d L_alpha / d log_alpha}, as the continuous learner's.
 * get_action: Categorical(actor(s)).sample(), epsilon ignored (Choose_Action2 -> get_action ignores it).  On the device: one
 * uniform u in [0, 1) per row -- Philox word 0 on the learner's act-call counter, the stream uavrl_sac_act draws its noise on
 * (key seed ^ 0x5AC5, trainer g: seed + g), or an injected tape -- then the smallest k with u sum(p) < p_0 + ... + p_k
 * (summed left to right in fp32), or, if rounding leaves none, the last k with p_k > 0.  The deterministic policy
 * (mean_action = 1) is argmax p, the lowest index on ties.
 * Limits: act_dim = A in [2, 31] (one 32-column head plane), obs_dim a multiple of 4 in [4, 128], hidden in [1, 128], and every
 * kernel's shared memory at most 227 KB (the shipped 100-64-64-27 fits: uavrl_sac_smem_bytes reports the four discrete
 * kernels, target, critic update, actor update, get_action).  Refused with UAVRL_ERR_INVALID before anything is allocated.
 * What changes against the continuous learner:
 *   - roles, uavrl_sac_param_count, set/get_params, alpha, scalars, grouped trainers and the actor aggregation keep their
 *     meaning; the flat layouts are actor = fc1, fc2, fc3 and critic = fc1, fc2, fc3 (state_dict order);
 *   - uavrl_sac_update_batch / uavrl_sac_critic_grads_batch take a_dev as int32 [B] action indices; the ring holds int32
 *     actions and uavrl_sac_replay_gather writes a_host as int32 [n];
 *   - uavrl_sac_act_discrete acts (below); uavrl_sac_act and uavrl_sac_act_mean are refused (UAVRL_ERR_INVALID);
 *   - uavrl_sac_train_run acts with the discrete kernel and steps the env with UAVRL_ACT_DISCRETE27, and refuses
 *     (UAVRL_ERR_INVALID) a learner whose act_dim is not 27; uavrl_sac_eval_run does the same, mean_action selecting argmax;
 *   - refused with UAVRL_ERR_INVALID (the reference's discrete update() has no importance weights; a data-parallel discrete
 *     update is not provided): prioritised replay (uavrl_sac_per_enable, uavrl_sac_update_batch_per) and every data-parallel
 *     call (uavrl_sac_comm_init / _connect, uavrl_sac_update_replay_dp, uavrl_sac_train_run_dp, the split calls). */
/* get_action of a discrete learner on n rows in G equal blocks: actions_dev int32 [n].  u_dev (may be NULL) [n] injects the
 * uniforms; else Philox on the act-call counter.  Either way the call advances the counter by one, as uavrl_sac_act does.  mean_action = 1: argmax p, drawing nothing and leaving
 * the counter as it is.  Refused on a continuous learner. */
int uavrl_sac_act_discrete(uavrl_sac *s, const float *obs_dev, int32_t n, const float *u_dev, int32_t mean_action, int32_t *actions_dev,
                           void *stream);
/* SAC_Trainer.update (:317-379, continuous) on an explicit batch: s [B][obs], a [B][2], r [B], s2 [B][obs], d [B];
 * eps_next / eps_cur [B][2] = noise of the two actor evaluations (NULL = Philox); losses_dev (optional) [4] =
 * {actor_loss, critic_1_loss, critic_2_loss, d alpha_loss / d log_alpha}. */
int uavrl_sac_update_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                           const float *d_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev, void *stream);
/* The lockstep replay ring (lockstep_envs > 0): uavrl_sac_replay_size = transitions held; uavrl_sac_replay_gather reads n of
 * them back by logical index (0 = oldest; k -> frame k / N, env k % N) into host arrays s/s2 [n][obs], a [n][2], r [n], d [n]. */
int64_t uavrl_sac_replay_size(const uavrl_sac *s);
int uavrl_sac_replay_gather(uavrl_sac *s, int32_t n, const int64_t *logical_idx_host, float *s_host, float *a_host, float *r_host,
                            float *s2_host, uint8_t *d_host);
/* One SAC_Trainer.update sampled from the lockstep ring, as uavrl_sac_train_run performs it: epoch += 1, skipped while the ring
 * holds <= batch_size transitions.  idx_tape_dev [batch_size] injects logical indices (NULL = Philox sampling); eps_next / eps_cur
 * and losses_dev as in uavrl_sac_update_batch. */
int uavrl_sac_update_replay(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev,
                            void *stream);
/* PathPlan_City.run_thread_OffPolicy + update with the SAC trainer and the reference's continuous step, N envs in lockstep:
 * the iteration of uavrl_train_run with one SAC update per iteration when do_update (stats_host->last_loss: the mean actor
 * loss over trainers).  Refused before anything is enqueued, leaving env, ring, parameters and counters untouched:
 * lockstep_envs != env.n_envs or no ring, obs_dim != 100 (the env step writes 100-float observations into the ring) or env and
 * learner on different devices (UAVRL_ERR_INVALID, as uavrl_train_run); no uavrl_env_reset (UAVRL_ERR_STATE). */
int uavrl_sac_train_run(uavrl_env *env, uavrl_sac *s, int32_t n_iters, int32_t do_update, uavrl_train_stats *stats_host, void *stream);

/* Prioritised replay for SAC (IsPriority_Replay = 1; SAC_Trainer.update :336-352, BaseClass/replay_buffer.py:57-223): one
 * SumTree per trainer over its own slots of the lockstep ring, the trees and rules of the uavrl_per_* block.  As written, the
 * reference's branch cannot run: is_weights * critic_loss is a [B,1] tensor that .backward() refuses (not a scalar), the critics'
 * action_dim = 2 outputs hand batch_update [B,2] errors that one SumTree leaf cannot hold, and its float tree_idx cannot index.
 * So this port states the semantics, taking the only readings that run and agree with the Q-network learner:
 *   - critic losses  L_k = mean over B x 2 of w_b (Q_k[b][j] - y[b][j])^2, k = 1, 2, with w_b the sample's importance weight
 *     (ReplayTree.sample2, normalised by the batch maximum of its trainer); the reported critic losses are these;
 *   - priority error e_b = 0.5f * (|m_0 - y_0| + |m_1 - y_1|), m_j = fminf(Q1[b][j], Q2[b][j]), float32 in that order -- the mean
 *     over the action columns, the reference's |min(Q1, Q2) - y| for action_dim = 1 -- from the critics BEFORE this update's
 *     step; it goes back through batch_update (clip): p = min(e + eps, err_upper)^alpha;
 *   - the actor loss, the alpha loss, the TD target and the soft update take no weights (:361-379);
 *   - a newly committed ring frame gets the error-less push priority (0 + eps)^alpha, the frame it drops 0.
 * Once enabled, every update that samples the ring without an injected idx_tape_dev (uavrl_sac_update_replay, uavrl_sac_train_run,
 * uavrl_sac_update_replay_dp, uavrl_sac_train_run_dp, uavrl_sac_critic_grads_replay) draws batch_size rows per trainer from the
 * trees (keyed as uavrl_per_sample), runs the critic leg weighted, writes every e_b back once the critic kernel has run, and
 * takes the actor leg on the same rows.  Trainer g of a grouped learner computes what a stand-alone learner with seed + g,
 * replay_capacity / G and lockstep_envs / G computes, its tree and beta included; data-parallel ranks keep trees of their own.
 *
 * uavrl_sac_per_enable: one call for every trainer count (the ring's slot numbering is the same for any G); negative
 * hyper-parameters take the reference's defaults.  Refused: no ring (lockstep_envs == 0; UAVRL_ERR_STATE), already enabled
 * or a transition already stored (UAVRL_ERR_STATE), more than 4 194 304 slots per tree (UAVRL_ERR_INVALID).
 * uavrl_sac_per_sample / _set_errors / _set_priorities / _get: the arguments, [G][...] shapes, trainer-local slots and refusals
 * of uavrl_per_sample / _set_errors / _set_priorities / _get (UAVRL_ERR_INVALID "prioritised replay not enabled" before
 * uavrl_sac_per_enable); uavrl_sac_per_sample is also refused (UAVRL_ERR_STATE) while a split update waits for its next phase.
 * uavrl_sac_update_batch_per: uavrl_sac_update_batch with importance weights is_weights_dev [B] (required; block g of G B / G
 * for trainer g) in the critic losses and e_b written to abs_err_out_dev [B] (may be NULL); it does not touch the trees. */
int uavrl_sac_per_enable(uavrl_sac *s, double alpha, double beta0, double beta_inc, double eps, double err_upper);
int uavrl_sac_per_sample(uavrl_sac *s, int32_t B, const double *u_tape_dev, int32_t *slots_out_dev, float *weights_out_dev, void *stream);
int uavrl_sac_per_set_errors(uavrl_sac *s, int32_t n, const int32_t *slots_dev, const float *abs_err_dev, int32_t clip, void *stream);
int uavrl_sac_per_set_priorities(uavrl_sac *s, int32_t n, const int32_t *slots_dev, const double *prio_dev, void *stream);
int uavrl_sac_per_get(uavrl_sac *s, double *leaves_host, double *total_out, double *beta_out);
int uavrl_sac_update_batch_per(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                               const float *d_dev, const float *is_weights_dev, float *abs_err_out_dev, const float *eps_next_dev,
                               const float *eps_cur_dev, float *losses_dev, void *stream);

/* Data-parallel SAC (one learner per GPU, each rank sampling batch_size rows from its own ring shard; global_batch =
 * batch_size x world).  The actor loss is taken on the UPDATED critics, so an update makes two exchanges: both critics'
 * gradients with the two critic squared-error sums, then -- after the critics' Adam step on every rank -- the actor's
 * gradient with the actor-loss and entropy sums.  All losses, the alpha step and the soft target update then use the
 * global sums over global_batch x 2 entries, and every rank holds bit-identical networks, Adam moments, alpha triple, epoch
 * and adam_step.  Each rank keeps its own seed, so its sampling keys and reparameterisation noise are its own.  With world =
 * 1 and global_batch = batch_size an update equals uavrl_sac_update_replay bit for bit (roles 11-13 hold 0 + g: a -0
 * gradient entry reads +0).
 *
 * Fused form (no NCCL): uavrl_sac_comm_init allocates this rank's receive buffer recv[2][world][max(2 Pc + 2, Pa + 2)] of
 * 8-byte words and writes UAVRL_SAC_COMM_HANDLE_BYTES bytes: its CUDA IPC handle followed by this device's PCI bus id;
 * uavrl_sac_comm_connect takes every rank's record ([world][UAVRL_SAC_COMM_HANDLE_BYTES] bytes) and refuses
 * (UAVRL_ERR_INVALID) two ranks on one device, whose exchange could never complete.  uavrl_sac_update_replay_dp is one
 * update from the ring through the two exchanges of uavrl_learner_update_dp's kernel (one word {tag : value} per value,
 * pushed to every rank, summed in rank order); a rank's exchange waits until every other rank's words arrive.
 *
 * Split form (e.g. NCCL, or a caller holding explicit batches), four calls in this order:
 *   uavrl_sac_critic_grads_replay / _batch  epoch += 1; sample from the ring (idx_tape_dev as in uavrl_sac_update_replay) or
 *                                           take B explicit rows (which must stay valid until the actor phase); write the
 *                                           critic exchange vector uavrl_sac_exchange_ptr(s, 0, &n): [grad critic_1 | grad
 *                                           critic_2 | critic-1, critic-2 squared-error sums], n = 2 Pc + 2;
 *   uavrl_sac_apply_critic_grads            after the caller summed that vector over the ranks: Adam on both critics;
 *   uavrl_sac_actor_grads                   the actor leg on the same rows (and the same ring contents) with eps_cur_dev;
 *                                           writes uavrl_sac_exchange_ptr(s, 1, &n): [grad actor | actor-loss sum,
 *                                           entropy sum], n = Pa + 2;
 *   uavrl_sac_apply_actor_grads             after the sum: the actor's Adam step, the alpha step, the soft target update and
 *                                           losses_dev [4] (global means).
 * Refused before the epoch counts, leaving parameters, moments, alpha, counters and ring untouched: a learner with several
 * trainers and global_batch <= 0 (UAVRL_ERR_INVALID); a call out of the order above, no ring or a ring holding <=
 * batch_size transitions for the ring forms, uavrl_sac_update_replay_dp before uavrl_sac_comm_connect (UAVRL_ERR_STATE). */
#define UAVRL_SAC_COMM_HANDLE_BYTES 128
int uavrl_sac_comm_init(uavrl_sac *s, int32_t rank, int32_t world, void *handle_out);
int uavrl_sac_comm_connect(uavrl_sac *s, const void *handles);
int uavrl_sac_update_replay_dp(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, const float *eps_cur_dev,
                               int32_t global_batch, float *losses_dev, void *stream);
int uavrl_sac_critic_grads_replay(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, int32_t global_batch, void *stream);
int uavrl_sac_critic_grads_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                                 const float *d_dev, const float *eps_next_dev, int32_t global_batch, void *stream);
int uavrl_sac_apply_critic_grads(uavrl_sac *s, void *stream);
int uavrl_sac_actor_grads(uavrl_sac *s, const float *eps_cur_dev, void *stream);
int uavrl_sac_apply_actor_grads(uavrl_sac *s, float *losses_dev, void *stream);
/* phase 0: the critic exchange vector, 1: the actor's; *len_out (may be NULL) receives its length in floats.  Device memory
 * owned by the learner; NULL for another phase. */
float *uavrl_sac_exchange_ptr(uavrl_sac *s, int32_t phase, int64_t *len_out);
/* Data-parallel form of uavrl_sac_train_run (after uavrl_sac_comm_connect): every iteration ends with one
 * uavrl_sac_update_replay_dp on this rank's ring.  Refused before anything is enqueued, leaving env, ring, parameters and
 * counters untouched: global_batch <= 0, a learner with several trainers, and what uavrl_sac_train_run refuses
 * (UAVRL_ERR_INVALID); no uavrl_sac_comm_connect, no uavrl_env_reset, or a ring that would hold <= batch_size transitions
 * at the first update (UAVRL_ERR_STATE: warm it up with uavrl_sac_train_run first). */
int uavrl_sac_train_run_dp(uavrl_env *env, uavrl_sac *s, int32_t n_iters, int32_t global_batch, void *stream);

/* Data-parallel form of uavrl_train_run (after uavrl_learner_comm_connect): every iteration ends with
 * uavrl_learner_update_dp on this rank's replay shard; global_batch = batch_size x world.  Refused before anything is
 * enqueued, leaving env, ring, parameters and counters untouched: global_batch <= 0, a grouped learner, lockstep_envs !=
 * env.n_envs, in_dim != 100 or env and learner on different devices (UAVRL_ERR_INVALID, as uavrl_train_run); no
 * uavrl_learner_comm_connect, no uavrl_env_reset, or a ring that would hold <= batch_size transitions at the first
 * update (UAVRL_ERR_STATE: warm it up with uavrl_train_run first; the count never shrinks, so every later update runs). */
int uavrl_train_run_dp(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t global_batch, void *stream);

/* The same loop with a CUDA event recorded on `stream` before/after every kernel: ms_out[6] receives the
 * summed device time of {act, env_step, td_target, fwd_bwd, weight_grad, reduce_adam} over the n_iters
 * iterations (bench.py's roofline pass; on the CUDA-core path td_target and weight_grad are 0 because
 * fwd_bwd does everything; event gaps make the loop slower, never use it for throughput).  Refused before anything is
 * enqueued: in_dim != 100 or env and learner on different devices (UAVRL_ERR_INVALID, as uavrl_train_run), a pair that
 * has never run uavrl_train_run or a ring that would hold <= batch_size transitions per trainer at the first update
 * (UAVRL_ERR_STATE, as uavrl_train_run_dp). */
int uavrl_train_profile(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, float *ms_out, void *stream);

/* ---- prioritised experience replay (SURVEY.md 8f-3) ------------------------------------------------------------
 * Replaces SumTree + ReplayTree (BaseClass/replay_buffer.py:57-223): priorities per replay slot, stratified sampling
 * over `batch` equal segments of int(total), importance weights (n p / total)^-beta / max, beta += beta_inc per
 * sampling call (capped at 1), batch_update with (min(|err| + eps, err_upper))^alpha.  Arguments < 0 take the
 * reference's constants (alpha 0.6, beta 0.4, beta_inc 0.001, eps 0.01, err_upper 1).  Enable before the first
 * transition is stored.  Once enabled:
 *   - uavrl_replay_push / the lockstep loops give new transitions the priority of ReplayTree.push with error 0;
 *   - uavrl_learner_update / uavrl_train_run sample through it, minimise mean(w_i (Q - y)^2) and write
 *     |Q - y| back with the batch_update rule.  (The reference multiplies the weights into the already averaged loss,
 *     SAC_Trainer.py:348-352, which cannot be back-propagated; the per-sample form is the documented deviation.)
 * uavrl_per_sample = ReplayTree.sample2 (:186-213): physical slot indices (tree index = slot + capacity - 1) and
 * weights; u_tape_dev (optional, [batch] doubles in [0,1)) replaces the uniform draws.  uavrl_per_set_errors:
 * clip = 0 is ReplayTree.push's rule (:152-154), clip = 1 batch_update's (:216-223).  uavrl_per_set_priorities is
 * SumTree.update with explicit values.  uavrl_per_get copies the leaves [slots] to the host.
 *
 * uavrl_per_enable_trainers: the same for a learner with G >= 1 trainers (identical to uavrl_per_enable when G = 1; G > 1 needs
 * the lockstep ring).  Trainer g gets its own tree over its own transitions, as each reference Trainer owns its ReplayTree, and
 * computes bit for bit what a stand-alone learner with prioritised replay, seed + g and Ng = lockstep_envs / G envs computes.
 * Slots are trainer-local: transition (ring frame f, env e) of trainer g's block is slot j = f Ng + (e - g Ng), in
 * [0, cap_g), cap_g = ring_frames Ng (the numbering of a stand-alone learner over Ng envs).  cap_g <= 4194304.  Refused after
 * the first stored transition.  Afterwards, on a grouped learner:
 *   - uavrl_per_sample: batch is per trainer; u_tape_dev [G][batch]; slots / weights out [G][batch], each row normalised by
 *     that trainer's own maximum weight, n = that trainer's transition count; trainer g's draws are keyed by seed + g;
 *   - uavrl_per_set_errors / uavrl_per_set_priorities: n is per trainer; slots and values [G][n];
 *   - uavrl_per_get: leaves [G][cap_g], total_out [G], beta (shared: the trainers sample in lockstep);
 *   - uavrl_learner_update / uavrl_train_run sample every trainer from its own tree and write |Q - y| back into it. */
int uavrl_per_enable(uavrl_learner *l, double alpha, double beta0, double beta_inc, double eps, double err_upper);
int uavrl_per_enable_trainers(uavrl_learner *l, double alpha, double beta0, double beta_inc, double eps, double err_upper);
int uavrl_per_sample(uavrl_learner *l, int32_t batch, const double *u_tape_dev, int32_t *slots_out_dev,
                     float *weights_out_dev, void *stream);
int uavrl_per_set_errors(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const float *abs_err_dev, int32_t clip,
                         void *stream);
int uavrl_per_set_priorities(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const double *priorities_dev,
                             void *stream);
int uavrl_per_get(uavrl_learner *l, double *leaves_host, double *total_out, double *beta_out);
/* Trainer.update(transition_dict) with 'weights' (and |TD error| back for batch_update): uavrl_learner_update_batch
 * with per-sample importance weights in the loss; is_weights_dev / abs_err_out_dev may be NULL. */
int uavrl_learner_update_batch_per(uavrl_learner *l, int32_t batch, const float *obs_dev, const int32_t *act_dev,
                                   const float *rew_dev, const float *next_obs_dev, const float *done_dev,
                                   const float *is_weights_dev, float *abs_err_out_dev, float *loss_dev, void *stream);

/* ---- policy evaluation (greedy episodes over a held-out scenario suite) --------------------------------------------
 * The reference leaves its evaluation hooks as stubs (PathPlan_City.Evaluation_Action, Sim) and never advances
 * UAV.Testing_time; it only counts successes while training, under exploration and with the replay filling.  These calls run
 * a learner's policy on its own, one uavrl_episode_record per episode:
 *   - the suite is pool scenarios first_scenario + k (mod P), k in [0, n_episodes); env e starts on position e and after its
 *     j-th episode takes position (j + 1) n_envs + e; an env with no position left parks: it is not stepped again, writes no
 *     record and adds to no statistic (envs e >= n_episodes are never reset or stepped).  The env's auto_reset, reset stride
 *     and records are its own again afterwards; its state is the evaluation's final state;
 *   - actions: uavrl_eval_run acts greedily (uavrl_learner_act with is_train = 0) and leaves the act-call counter as it was;
 *     uavrl_sac_eval_run samples as SAC_Trainer.get_action does (Trainer/SAC_Trainer.py:444-448), with noise keyed by the
 *     learner seed (trainer g: seed + g), first_scenario and the iteration, on counters no training draw uses -- or, with
 *     mean_action = 1, takes tanh(mu) bound (uavrl_sac_act_mean).  Env block g acts with trainer g; n_envs must be a multiple
 *     of the trainer count.  Nothing of the learner changes: parameters, moments, alpha, counters, ring and trees;
 *   - the loop stops once every suite episode has its record, or after max_iters iterations (0: ceil(n / n_envs) K max_step,
 *     which every suite episode ends within).  It reads the record count every 64 iterations, so iterations may run past
 *     the last record (parked envs do nothing);
 *   - records_host (may be NULL) receives [n_episodes] records in suite order (record k = position k; outcome 0: unfinished);
 *     stats_host (may be NULL) the iterations run, the records written and the episodes left unfinished.
 * Refused before anything is enqueued: n_episodes or max_iters < 0, learner input width != 100, env and learner on different
 * devices, n_envs not a multiple of the trainer count, a Q-network without 27 actions or mean_action not 0 / 1
 * (UAVRL_ERR_INVALID); no pool (UAVRL_ERR_STATE).  Synchronises `stream`. */
typedef struct {
    int64_t iterations, records, unfinished;
} uavrl_eval_stats;
int uavrl_eval_run(uavrl_env *env, uavrl_learner *l, int32_t first_scenario, int32_t n_episodes, int64_t max_iters,
                   uavrl_episode_record *records_host, uavrl_eval_stats *stats_host, void *stream);
int uavrl_sac_eval_run(uavrl_env *env, uavrl_sac *s, int32_t first_scenario, int32_t n_episodes, int32_t mean_action,
                       int64_t max_iters, uavrl_episode_record *records_host, uavrl_eval_stats *stats_host, void *stream);
/* The SAC policy's mean action tanh(mu) bound for n rows in G equal blocks (PolicyNetContinuous_SAC.forward without noise);
 * draws nothing and leaves the act-call counter as it is. */
int uavrl_sac_act_mean(uavrl_sac *s, const float *obs_dev, int32_t n, float *actions_dev, void *stream);

const char *uavrl_last_error(void);
const char *uavrl_version(void);
/* number of kernel launches issued by this library in the calling process since load (bench.py) */
int64_t uavrl_launch_count(void);
/* Programmatic dependent launch inside the lockstep loops (each kernel's prologue overlaps its predecessor's
 * tail; results are unchanged).  Process-wide switch, default 1; 0 launches every kernel fully serialised. */
int uavrl_set_pdl(int32_t on);
/* Test hook for the out-of-memory paths.  n >= 0: of the library's device allocations from now on, the first n succeed and
 * the next one fails as an exhausted cudaMalloc does (UAVRL_ERR_CUDA, "out of memory"); the hook then turns itself off.
 * n = -1 (the default) turns it off.  Process-wide. */
int uavrl_test_fail_alloc(int32_t n);
/* Kept for ABI compatibility; 0 only.  The lockstep loops launch get_action and Move_Agent as two kernels.  on = 0 returns 0;
 * any other value returns UAVRL_ERR_INVALID (the fused variant was removed). */
int uavrl_set_fuse_act_env(int32_t on);
/* Kept for ABI compatibility; 0 only.  The optimiser step runs as its own kernel behind the weight-gradient kernel.  on = 0
 * returns 0; any other value returns UAVRL_ERR_INVALID (the fused variant was removed). */
int uavrl_set_fuse_dw_adam(int32_t on);
/* Batches of at most 132 x 32 transitions (132 x 64 on 64-row tiles when the operands fit shared memory) on the tensor-core path: the TD-target forward pass(es) (target network on the next
 * states; double DQN: the local network first) run inside the training kernel, each CTA on the tile it then trains on
 * (weight images restaged in shared memory between the passes, y kept in shared memory) -- one launch instead of two or
 * three per update; the arithmetic is the stand-alone passes'.  Process-wide switch, default 1. */
int uavrl_set_fuse_td(int32_t on);
/* 1 if an update of `batch` transitions on this learner runs the TD-target pass(es) inside the training kernel (see above). */
int uavrl_learner_td_fused(const uavrl_learner *l, int32_t batch);
/* Which kernels an act / TD pass over n samples and an update of a batch of n run on this learner, with its current
 * tensor-core setting.  out[6]: [0] tensor-core act / TD pass, [1] tensor-core training kernel (0 = not used, the fp32
 * CUDA-core kernel runs; 1 = generic variant, runtime k-step chains; 2 = FIXED variant, compile-time chains); [2] rows per
 * tile of that act / TD pass, [3] rows per tile of that training kernel (0 when not used); [4] the TD-target pass(es) run
 * inside the training kernel; [5] the fp32 update kernel keeps both networks' weights in shared memory at once. */
int uavrl_learner_tc_route(const uavrl_learner *l, int32_t n, int32_t *out);

#ifdef __cplusplus
}
#endif
#endif /* UAVRL_H */
