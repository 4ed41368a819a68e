// env.cuh -- device-side view of a batch of UAV environments (SoA, fp64 state) + host handle.
#pragma once
#include "common.cuh"
#include "env_core.cuh"

#include <vector>

namespace uavrl {

constexpr int kEnvThreads = 128;       // warp 0 steps the CTA's envs; all 4 warps share their probes
// envs per CTA: 8 while the whole batch then fits ONE wave (4 CTAs of 128 threads per SM), so that the latency-bound fp64
// chains of a 4096-env step spread over 512 CTAs instead of 128; 32 above, where 8 per CTA would need several waves
constexpr int kEnvsPerBlockLarge = 32, kEnvsPerBlockSmall = 8;
inline int small_batch_envs() { return 4 * num_sms() * kEnvsPerBlockSmall; }
constexpr int kMaxCyl = 64;            // candidate sets are 64-bit masks

// Everything a kernel needs, passed by value.
struct EnvDev {
    EnvConst k;
    int32_t n, K, P;
    int32_t auto_reset;
    int32_t reset_stride;               // scenario advance of an env's auto-reset: n, or the full batch's n for a shard of it
    double cull_w;                     // half-width of the probe window incl. one step of motion
    const Cyl *cyl;
    // per-env state, structure of arrays
    double *px, *py, *pz, *vx, *vy, *V, *score, *total, *path_len, *gx, *gy, *gz, *rew64, *theta;
    int32_t *step, *cursor, *n_sub, *scen;
    uint8_t *done, *alias;
    // scenario pool (read-only during stepping)
    const double *pool_start, *pool_goal, *pool_v0, *pool_sub;
    const int32_t *pool_nsub;
    const uint8_t *pool_alias;
    // running statistics: [0] env steps, [1] episodes ended, [2] collisions ; sum_reward separately
    unsigned long long *stat_counts;
    double *stat_reward;
    // optional models (uavrl_env_set_extras); extras = bit mask kExtra*
    int32_t extras;
    PowerConst pw;                      // energy: Calc_Fly_Power constants
    double *energy;                     // [n] accumulated over the episode in progress
    const ApfObs *apf_obs;              // APF: every obstacle with its velocity (device)
    double *sub_env;                    // APF: per-env sub-goal queues [n][K][3] (shifted every step)
    double *path_buf;                   // track: [2][track_n][track_cap][3]
    int32_t *path_n;                    // [2][track_n] points recorded (buffer 0/1)
    int32_t *path_cur;                  // [track_n] buffer holding the episode in progress
    int32_t track_n, track_cap;
    long long *trace;                   // debug (UAVRL_ENV_TRACE): CTA 0 / thread 0 stage timestamps
};
constexpr int kExtraEnergy = 1, kExtraApf = 2, kExtraTrack = 4, kExtraRecord = 8, kExtraMotion = 16;

// Moving obstacles (uavrl_env_set_motion): the device view the EXTRAS step takes as its own kernel argument.  The step reads
// O_t from rd and CTA 0 writes O_{t+1} to wr, the other buffer; the host flips the two after each launch.
struct EnvMotionDev {
    const MoveObs *rd;
    MoveObs *wr;                        // null for an observation (nothing advances)
    const double *dir;                  // [n_cyl][4][2]: cos, sin of calculate_angle(0, v) per motion_variant of v
    double len, width;
};

// The table's owner: two buffers of n_cyl rows, the APF directions, and what set_motion was given
struct EnvMotion {
    DevMem mem;
    MoveObs *buf[2] = { nullptr, nullptr };
    double *dir = nullptr;
    int cur = 0;                        // the buffer holding O_t
    int64_t steps = 0;                  // step calls since set_motion
    double reach = 0.0;                 // added to the cull half-width: the largest |vx|, |vy| plus a margin
    std::vector<double> v;              // [n_cyl][3] velocities as set (vz included)
    bool on = false;
    EnvMotionDev view(bool advance, double len, double width) const
    {
        return { buf[cur], advance ? buf[cur ^ 1] : nullptr, dir, len, width };
    }
};

// Per-CTA staging of the moving table (env_extras_kernel only): O_t as read, and the APF table at O_t
struct MotionSmem {
    MoveObs o[kMaxCyl];
    ApfObs apf[kMaxCyl];
};

// Episode records (uavrl_env_set_records): the device view the EXTRAS step takes as its own kernel argument, so EnvDev and the
// default step keep their layout.  Episode j of env e goes to slot j n + e; a slot at or beyond cap is counted as dropped.
// limit: suite positions of an evaluation (uavrl_eval_run): an env whose next position ord n + e is >= limit is parked -- the
// step leaves it alone; outside an evaluation limit is INT64_MAX and nothing parks.
struct EnvRecDev {
    uavrl_episode_record *rec;          // [cap]; outcome 0 marks a slot not written
    int64_t cap, limit;
    int32_t *ord, *steps, *coll;        // [n]: finished episodes since enable / clear; step calls and collisions of the episode
    unsigned long long *counts;         // [0] records written, [1] dropped
};

// The records' owner: device memory and view; on = false leaves the step's extras as they are.
struct EnvRecords {
    DevMem mem;
    EnvRecDev dev = { nullptr, 0, INT64_MAX, nullptr, nullptr, nullptr, nullptr };
    bool on = false;
};

}  // namespace uavrl

struct uavrl_env {
    uavrl_env_config cfg;
    uavrl::EnvDev d;
    // owners of the device arrays: cylinders, state columns and counters; the scenario pool; the extras; the host-step staging
    uavrl::DevMem mem, pool_mem, extras_mem, staging_mem;
    bool pool_set = false, reset_done = false;
    // staging for the host-buffer entry point, allocated (grow) by its first call: staging_n envs, 0 until then
    int32_t staging_n = 0;
    double *h_act_dev = nullptr;
    float *h_obs_dev = nullptr, *h_rew_dev = nullptr;
    uint8_t *h_flags_dev = nullptr;      // done | info | collision | ended, each [n]
    cudaStream_t own_stream = nullptr;
    bool extras_set = false;
    std::vector<double> base_z;          // building base heights (position.z), used by the APF distance only
    uavrl::EnvRecords records;           // uavrl_env_set_records; swapped out for its own by an evaluation (eval.cu)
    uavrl::EnvMotion motion;             // uavrl_env_set_motion
    std::vector<double> apf_v;           // [n_cyl][3] obstacle velocities of the APF model, when it is on
};

namespace uavrl {
// launched by env.cu, the fused training loops (train.cu) and the evaluation loop (eval.cu); with moving obstacles a launch
// advances the table, so the handle is not const
int launch_env_step(uavrl_env *env, int action_kind, const void *actions, float *obs, float *reward,
                    uint8_t *done, uint8_t *info, uint8_t *coll, uint8_t *ended, cudaStream_t st, bool pdl = false);
int launch_env_observe(const uavrl_env *env, float *obs, cudaStream_t st);
// env_reset_kernel over envs [0, n_reset) only (uavrl_env_reset: every env; an evaluation: the envs that have a suite position)
int launch_env_reset(uavrl_env *env, int first, int n_reset, cudaStream_t st);
// records (env.cu): allocate cap slots over the env's n rows (zeroed, stream-ordered on the env's device), and zero them again
int records_alloc(EnvRecords &r, int n, int64_t cap);
int records_clear(EnvRecords &r, int n, cudaStream_t st);
// the env counters around a training loop (uavrl_train_run, uavrl_sac_train_run): begin() reads them, end() fills `out` with
// what the loop added, all but last_loss, which each loop takes from its own losses.  Both synchronise `st`; nothing happens
// when out is null.
struct EnvStatsMark {
    unsigned long long c[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    double r = 0.0;
    int begin(const EnvDev &d, cudaStream_t st, const uavrl_train_stats *out);
    int end(const EnvDev &d, cudaStream_t st, int64_t updates, uavrl_train_stats *out) const;
};
// A scenario pool under construction (uavrl_env_set_pool fills it from the host, uavrl_env_generate_pool on the device):
// pool_alloc gives it P scenarios of K sub-goals, pool_install waits for the device and swaps it in for the env's pool.
struct PoolBuild { DevMem mem; double *start, *goal, *v0, *sub; int32_t *nsub; uint8_t *alias; };
int pool_alloc(PoolBuild &b, size_t P, size_t K);
int pool_install(uavrl_env *env, PoolBuild &b, int32_t P);
}  // namespace uavrl
