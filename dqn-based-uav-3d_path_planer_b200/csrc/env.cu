// env.cu -- batched PathPlan_City UAV step + observation kernel (sm_90a) and its C ABI.
//
// Replaces, for N independent UAV instances in lockstep:
//   BaseEnv.Move_Agent           BaseClass/BaseEnv.py:123-137
//   UAV.update_PathPlan          Agents/UAV.py:397-513
//   UAV.state_PathPlan           Agents/UAV.py:515-567   (80 Threaten_rate probes)
//   PathPlan_City.Threaten_rate  Envs/PathPlan_City.py:215-223
//   building.check_threaten      Obstacles/building.py:20-26
//   UAV.reset (draws supplied)   Agents/UAV.py:335-366
//
// Kernel shape (DESIGN.md section "env_step"):  one CTA = 32 envs, 128 threads.
//   phase 1  warp 0, one lane per env: SoA state -> registers (coalesced 8-byte columns), the
//            fp64 kinematics / reward / termination chain, optional auto-reset from the scenario
//            pool, state write-back, 20 real-valued observation entries -> smem tile, and the
//            exact-culling candidate mask (cylinders whose bounding box meets the probe window).
//   phase 2  all 4 warps: 32 x 80 occupancy probes, each against its env's candidate cylinders only
//            (typically 0-2 of the 26), sqrt-free guard-banded fast path with the reference's exact
//            `sqrt(s) < R` only inside the guard band -> results identical to the brute-force
//            80 x 26 loop.
//   phase 3  the CTA's 32 x 100 fp32 observation tile (12.8 KB, contiguous in HBM) is written
//            with 16-byte stores, fully coalesced; this is the only large traffic of the step.
#include <stdlib.h>
#include <stdio.h>
#include "env.cuh"
#include "env_block.cuh"

#include <math.h>
#include <string.h>
#include <cmath>
#include <vector>

namespace uavrl {

thread_local std::string g_last_error;
std::atomic<long long> g_launches{0};
std::atomic<int> g_pdl{1};
std::atomic<int> g_fail_alloc{-1};

template <bool DO_STEP, int EPB, bool EXTRAS = false>
__global__ void __launch_bounds__(kEnvThreads)
env_kernel(EnvDev d, int action_kind, const void *__restrict__ actions, float *__restrict__ obs,
           float *__restrict__ reward, uint8_t *__restrict__ done_out, uint8_t *__restrict__ info_out,
           uint8_t *__restrict__ coll_out, uint8_t *__restrict__ ended_out)
{
    static_assert(!EXTRAS, "the optional models run env_extras_kernel");
    __shared__ EnvSmem<EPB> sm;
    env_block<DO_STEP, EPB, kEnvThreads, true, (EPB < 32 ? EPB : 32), EXTRAS>(d, sm, blockIdx.x * EPB, threadIdx.x, action_kind, actions, obs,
                                                                              reward, done_out, info_out, coll_out, ended_out);
}

// The EXTRAS instantiation (uavrl_env_set_extras, uavrl_env_set_records): a kernel of its own, so that its records argument
// leaves the default kernels' parameters, and with them their code, as they are
template <bool DO_STEP, int EPB>
__global__ void __launch_bounds__(kEnvThreads)
env_extras_kernel(EnvDev d, int action_kind, const void *__restrict__ actions, float *__restrict__ obs,
                  float *__restrict__ reward, uint8_t *__restrict__ done_out, uint8_t *__restrict__ info_out,
                  uint8_t *__restrict__ coll_out, uint8_t *__restrict__ ended_out, EnvRecDev rec, EnvMotionDev mot)
{
    __shared__ EnvSmem<EPB> sm;
    __shared__ MotionSmem msm;
    env_block<DO_STEP, EPB, kEnvThreads, true, (EPB < 32 ? EPB : 32), true>(d, sm, blockIdx.x * EPB, threadIdx.x, action_kind, actions, obs,
                                                                            reward, done_out, info_out, coll_out, ended_out, &rec,
                                                                            &mot, &msm);
}

// uavrl_env_reset on envs [0, n_reset): the env's first scenario first + e; with records on, its episode counters restart
__global__ void env_reset_kernel(EnvDev d, int first, int n_reset, EnvRecDev rec)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= d.n || e >= n_reset) return;
    if (d.extras & kExtraRecord) { rec.steps[e] = 0; rec.coll[e] = 0; }
    const int scen = (int)(((long long)first + e) % d.P);
    EnvRegs s;
    load_scenario(d, scen, s);
    d.scen[e] = scen;
    d.px[e] = s.px; d.py[e] = s.py; d.pz[e] = s.pz;
    d.vx[e] = s.vx; d.vy[e] = s.vy; d.V[e] = s.V; d.theta[e] = s.theta;
    d.gx[e] = s.gx; d.gy[e] = s.gy; d.gz[e] = s.gz;
    d.score[e] = 0.0; d.total[e] = 0.0; d.path_len[e] = 0.0; d.rew64[e] = 0.0;
    d.step[e] = 0; d.cursor[e] = 0; d.n_sub[e] = s.n_sub;
    d.done[e] = 0; d.alias[e] = (uint8_t)s.alias;
    if (d.extras & kExtraEnergy) d.energy[e] = 0.0;
    if ((d.extras & kExtraTrack) && e < d.track_n) { d.path_cur[e] = 0; d.path_n[e] = 0; d.path_n[d.track_n + e] = 0; }
    if (d.extras & kExtraApf) {                                  // the env's own copy of the scenario's sub-goal queue
        const double *src = d.pool_sub + (size_t)scen * d.K * 3;
        double *dst = d.sub_env + (size_t)e * d.K * 3;
        for (int i = 0; i < d.K * 3; ++i) dst[i] = src[i];
    }
}

__global__ void env_theta_kernel(EnvDev d)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < d.n) d.theta[e] = angle_xy(d.vx[e], d.vy[e]);
}

// moved: the current moving table (uavrl_env_set_motion), or null for the cylinders as created
__global__ void threat_kernel(EnvDev d, int n, const double *__restrict__ pts, uint8_t *__restrict__ out, const MoveObs *moved)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    int hit = out_of_bounds(d.k, x, y, z);
    for (int c = 0; c < d.k.n_cyl && !hit; ++c) {
        Cyl cy = d.cyl[c];
        if (moved) { cy.cx = moved[c].x; cy.cy = moved[c].y; }
        hit = cyl_hit(cy, x, y, z);
    }
    out[i] = (uint8_t)hit;
}

int launch_env_step(uavrl_env *env, int action_kind, const void *actions, float *obs, float *reward,
                    uint8_t *done, uint8_t *info, uint8_t *coll, uint8_t *ended, cudaStream_t st, bool pdl)
{
    EnvDev d = env->d;
    const EnvRecDev &rec = env->records.dev;
    static const bool trace_on = getenv("UAVRL_ENV_TRACE") != nullptr;
    static DevMem tr_mem;
    static long long *tr = nullptr;
    static int n_traced = 0;
    if (trace_on) {
        if (!tr) { if (int rc = tr_mem.alloc(tr, 16)) return rc; }
        else if (++n_traced % 64 == 0) {                         // print the PREVIOUS launch's stamps every 64 launches
            long long h[16];
            UAVRL_CUDA(cudaStreamSynchronize(st));
            UAVRL_CUDA(cudaMemcpy(h, tr, sizeof(h), cudaMemcpyDeviceToHost));
            fprintf(stderr, "[env_trace] n=%d cycles since start:", d.n);
            for (int i = 1; i < 12; ++i) fprintf(stderr, " [%d]=%lld", i, h[i] - h[0]);
            fprintf(stderr, "\n");
        }
        d.trace = tr;
    }
    if (d.extras) {                                              // optional models: the EXTRAS instantiation (never inside a PDL chain)
        const int blocks = (d.n + kEnvsPerBlockSmall - 1) / kEnvsPerBlockSmall;
        EnvMotion &mo = env->motion;
        const EnvMotionDev mv = mo.view(true, env->cfg.len, env->cfg.width);
        // a candidate mask must also hold every cylinder that moves into the probe window during this step
        if (mo.on) d.cull_w += mo.reach;
        UAVRL_CUDA(launch_kernel(env_extras_kernel<true, kEnvsPerBlockSmall>, dim3(blocks), dim3(kEnvThreads), 0, st, pdl, d, action_kind, actions, obs,
                                 reward, done, info, coll, ended, rec, mv));
        if (mo.on) { mo.cur ^= 1; mo.steps += 1; }             // the launch succeeded: O_{t+1} is the table from now on
    } else if (d.n <= small_batch_envs()) {
        const int blocks = (d.n + kEnvsPerBlockSmall - 1) / kEnvsPerBlockSmall;
        UAVRL_CUDA(launch_kernel(env_kernel<true, kEnvsPerBlockSmall>, dim3(blocks), dim3(kEnvThreads), 0, st, pdl, d, action_kind, actions, obs,
                                 reward, done, info, coll, ended));
    } else {
        const int blocks = (d.n + kEnvsPerBlockLarge - 1) / kEnvsPerBlockLarge;
        UAVRL_CUDA(launch_kernel(env_kernel<true, kEnvsPerBlockLarge>, dim3(blocks), dim3(kEnvThreads), 0, st, pdl, d, action_kind, actions, obs,
                                 reward, done, info, coll, ended));
    }
    UAVRL_LAUNCHED();
    return 0;
}

int launch_env_observe(const uavrl_env *env, float *obs, cudaStream_t st)
{
    const EnvDev &d = env->d;
    const EnvRecDev &rec = env->records.dev;
    const int blocks = (d.n + kEnvsPerBlockLarge - 1) / kEnvsPerBlockLarge;
    const EnvMotionDev mv = env->motion.view(false, env->cfg.len, env->cfg.width);
    if (d.extras) env_extras_kernel<false, kEnvsPerBlockLarge><<<blocks, kEnvThreads, 0, st>>>(d, 0, nullptr, obs, nullptr, nullptr, nullptr, nullptr, nullptr, rec, mv);
    else env_kernel<false, kEnvsPerBlockLarge><<<blocks, kEnvThreads, 0, st>>>(d, 0, nullptr, obs, nullptr, nullptr, nullptr, nullptr, nullptr);
    UAVRL_LAUNCHED();
    return 0;
}

int launch_env_reset(uavrl_env *env, int first, int n_reset, cudaStream_t st)
{
    const int threads = 128, blocks = (env->d.n + threads - 1) / threads;
    env_reset_kernel<<<blocks, threads, 0, st>>>(env->d, first, n_reset, env->records.dev);
    UAVRL_LAUNCHED();
    env->reset_done = true;
    return 0;
}

int records_alloc(EnvRecords &r, int n, int64_t cap)
{
    EnvRecDev v = { nullptr, cap, INT64_MAX, nullptr, nullptr, nullptr, nullptr };
    int rc;
    if ((rc = r.mem.alloc(v.rec, (size_t)cap)) || (rc = r.mem.alloc(v.ord, (size_t)n)) || (rc = r.mem.alloc(v.steps, (size_t)n)) ||
        (rc = r.mem.alloc(v.coll, (size_t)n)) || (rc = r.mem.alloc(v.counts, 2)))
        return rc;
    r.dev = v;
    r.on = true;
    return 0;
}

// empties the slots and counts and restarts the ordinals; the episodes in progress keep their step and collision counts
int records_clear(EnvRecords &r, int n, cudaStream_t st)
{
    UAVRL_CUDA(cudaMemsetAsync(r.dev.rec, 0, (size_t)r.dev.cap * sizeof(uavrl_episode_record), st));
    UAVRL_CUDA(cudaMemsetAsync(r.dev.ord, 0, (size_t)n * 4, st));
    UAVRL_CUDA(cudaMemsetAsync(r.dev.counts, 0, 2 * sizeof(unsigned long long), st));
    return 0;
}

int EnvStatsMark::begin(const EnvDev &d, cudaStream_t st, const uavrl_train_stats *out)
{
    if (!out) return 0;
    UAVRL_CUDA(cudaStreamSynchronize(st));
    UAVRL_CUDA(cudaMemcpy(c, d.stat_counts, sizeof(c), cudaMemcpyDeviceToHost));
    UAVRL_CUDA(cudaMemcpy(&r, d.stat_reward, sizeof(r), cudaMemcpyDeviceToHost));
    return 0;
}

int EnvStatsMark::end(const EnvDev &d, cudaStream_t st, int64_t updates, uavrl_train_stats *out) const
{
    if (!out) return 0;
    UAVRL_CUDA(cudaStreamSynchronize(st));
    unsigned long long c1[8]; double r1;
    UAVRL_CUDA(cudaMemcpy(c1, d.stat_counts, sizeof(c1), cudaMemcpyDeviceToHost));
    UAVRL_CUDA(cudaMemcpy(&r1, d.stat_reward, sizeof(r1), cudaMemcpyDeviceToHost));
    out->env_steps = (int64_t)(c1[0] - c[0]);
    out->episodes_ended = (int64_t)(c1[1] - c[1]);
    out->collisions = (int64_t)(c1[2] - c[2]);
    out->n_success = (int64_t)(c1[3] - c[3]);
    out->n_lose = (int64_t)(c1[4] - c[4]);
    out->sum_reward = r1 - r;
    out->updates = updates;
    return 0;
}

}  // namespace uavrl

namespace uavrl {
int pool_alloc(PoolBuild &b, size_t P, size_t K)
{
    int rc;
    if ((rc = b.mem.alloc(b.start, P * 3, false)) || (rc = b.mem.alloc(b.goal, P * 3, false)) || (rc = b.mem.alloc(b.v0, P * 3, false)) ||
        (rc = b.mem.alloc(b.sub, P * K * 3, false)) || (rc = b.mem.alloc(b.nsub, P, false)) || (rc = b.mem.alloc(b.alias, P, false)))
        return rc;
    return 0;
}

int pool_install(uavrl_env *env, PoolBuild &b, int32_t P)
{
    UAVRL_CUDA(cudaDeviceSynchronize());            // nothing may still read the pool being replaced
    EnvDev &d = env->d;
    env->pool_mem = std::move(b.mem);
    d.pool_start = b.start; d.pool_goal = b.goal; d.pool_v0 = b.v0; d.pool_sub = b.sub; d.pool_nsub = b.nsub; d.pool_alias = b.alias;
    d.P = P; env->pool_set = true; env->reset_done = false;
    return 0;
}

// everything uavrl_env_create builds; on failure the caller destroys the half-built handle
static int env_init(uavrl_env *env, const uavrl_env_config *cfg)
{
    env->cfg = *cfg;
    env->cfg.buildings_host = nullptr;
    EnvDev &d = env->d;
    memset(&d, 0, sizeof(d));
    d.k.width = cfg->width; d.k.h = cfg->h;
    d.k.max_v = cfg->max_v; d.k.min_v = cfg->min_v; d.k.steering = cfg->steering_angle;
    d.k.climb = cfg->climb_rate; d.k.max_step = cfg->max_step; d.k.n_cyl = cfg->n_buildings;
    d.n = cfg->n_envs; d.K = cfg->max_subgoals; d.P = 0; d.auto_reset = cfg->auto_reset; d.reset_stride = cfg->n_envs;
    d.cull_w = 20.0 + cfg->max_v + 0.5;

    std::vector<Cyl> cyl((size_t)(cfg->n_buildings > 0 ? cfg->n_buildings : 1));
    for (int i = 0; i < cfg->n_buildings; ++i) {
        const double *b = cfg->buildings_host + 5 * i;
        Cyl c;
        c.cx = b[0]; c.cy = b[1]; c.R = b[3]; c.H = b[4];      // b[2] = base z: only ever subtracted from itself
        env->base_z.push_back(b[2]);                           // (the APF distance is 3-D: it does see it)
        const double r2 = c.R * c.R;
        c.r2lo = r2 * (1.0 - 1e-12); c.r2hi = r2 * (1.0 + 1e-12);
        cyl[i] = c;
    }
    DevMem &m = env->mem;
    int rc;
    Cyl *dcyl = nullptr;
    if ((rc = m.alloc(dcyl, cyl.size(), false))) return rc;
    UAVRL_CUDA(cudaMemcpy(dcyl, cyl.data(), cyl.size() * sizeof(Cyl), cudaMemcpyHostToDevice));
    d.cyl = dcyl;

    const size_t n = (size_t)d.n;
    double **f64[] = { &d.px, &d.py, &d.pz, &d.vx, &d.vy, &d.V, &d.score, &d.total, &d.path_len,
                       &d.gx, &d.gy, &d.gz, &d.rew64, &d.theta };
    for (auto p : f64) if ((rc = m.alloc(*p, n))) return rc;
    int32_t **i32[] = { &d.step, &d.cursor, &d.n_sub, &d.scen };
    for (auto p : i32) if ((rc = m.alloc(*p, n))) return rc;
    if ((rc = m.alloc(d.done, n)) || (rc = m.alloc(d.alias, n)) || (rc = m.alloc(d.stat_counts, 8)) ||
        (rc = m.alloc(d.stat_reward, 2)))                      // [0] sum of rewards, [1] total flight energy (extras)
        return rc;
    UAVRL_CUDA(cudaStreamCreateWithFlags(&env->own_stream, cudaStreamNonBlocking));
    return 0;
}
}  // namespace uavrl

using namespace uavrl;

// ------------------------------------------------------------------------------------ C ABI
extern "C" {

const char *uavrl_last_error(void) { return g_last_error.c_str(); }
int uavrl_set_pdl(int32_t on) { g_pdl.store(on ? 1 : 0); return 0; }
int uavrl_test_fail_alloc(int32_t n) { g_fail_alloc.store(n >= 0 ? n : -1); return 0; }
const char *uavrl_version(void) { return "uavrl-b200 0.1 (sm_90a)"; }
int64_t uavrl_launch_count(void) { return (int64_t)g_launches.load(); }

int uavrl_env_create(const uavrl_env_config *cfg, uavrl_env **out)
{
    if (!cfg || !out) return fail(UAVRL_ERR_INVALID, "uavrl_env_create: null argument");
    if (cfg->n_envs <= 0 || cfg->max_subgoals <= 0) return fail(UAVRL_ERR_INVALID, "n_envs and max_subgoals must be > 0");
    if (cfg->n_buildings < 0 || cfg->n_buildings > kMaxCyl)
        return fail(UAVRL_ERR_INVALID, "n_buildings must be in [0,64] (candidate sets are 64-bit masks)");
    if (cfg->n_buildings > 0 && !cfg->buildings_host) return fail(UAVRL_ERR_INVALID, "buildings_host is null");
    if (cfg->max_step <= 0 || !(cfg->max_v > 0)) return fail(UAVRL_ERR_INVALID, "max_step and max_v must be > 0");
    // A negative speed level turns V_vector against the heading the step carries (UAV.py:414-416 recomputes it from
    // V_vector every step, the cached heading does not), so the discrete-27 speeds Min_V, (Min_V + Max_V) / 2 must be >= 0.
    if (!(cfg->min_v >= 0)) return fail(UAVRL_ERR_INVALID, "min_v must be >= 0: a negative speed reverses V_vector against the heading");
    // RRT.py:69-71 makes sub_goals[0] the UAV's own position object: a collision on the very first step moves that entry with
    // the UAV.  The kernel does not write the moved entry back to the queue -- immaterial while one step is shorter than the 7 m
    // sub-goal radius (the entry is popped on that same step; reference Max_V = 1), a divergence from the reference beyond it.
    if (!(cfg->max_v < 7.0)) return fail(UAVRL_ERR_INVALID, "max_v must be < 7 (sub-goal radius): larger steps are outside the validated model");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(UAVRL_ERR_CUDA, "no CUDA device: the UAV step has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg->device));

    uavrl_env *env = new uavrl_env();
    if (int rc = env_init(env, cfg)) { uavrl_env_destroy(env); return rc; }
    *out = env;
    return 0;
}

int uavrl_env_destroy(uavrl_env *env)
{
    if (!env) return 0;
    cudaSetDevice(env->cfg.device);
    if (env->own_stream) cudaStreamDestroy(env->own_stream);
    delete env;
    return 0;
}

int uavrl_env_set_pool(uavrl_env *env, int32_t P, const double *start, const double *goal,
                       const double *heading, const double *sub, const int32_t *n_sub, const uint8_t *alias0)
{
    if (!env || P <= 0 || !start || !goal || !heading || !sub || !n_sub)
        return fail(UAVRL_ERR_INVALID, "uavrl_env_set_pool: null/empty argument");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    EnvDev &d = env->d;
    for (int i = 0; i < P; ++i)
        if (n_sub[i] < 0 || n_sub[i] > d.K) return fail(UAVRL_ERR_INVALID, "n_sub exceeds max_subgoals");
    // UAV.py:344-348: V_vector = Max_V*(cos, sin)(heading); V = Calc_V().  Done on the host with libm so
    // the initial velocity is the reference's bit pattern.
    std::vector<double> v0((size_t)P * 3);
    std::vector<uint8_t> al((size_t)P, 1);
    for (int i = 0; i < P; ++i) {
        double vx = env->cfg.max_v * cos(heading[i]), vy = env->cfg.max_v * sin(heading[i]);
        double V = sqrt(vx * vx + vy * vy + 0.0);
        if (V > env->cfg.max_v) { vx = vx * (env->cfg.max_v / V); vy = vy * (env->cfg.max_v / V); V = env->cfg.max_v; }
        v0[3 * i] = vx; v0[3 * i + 1] = vy; v0[3 * i + 2] = V;
        if (alias0) al[i] = alias0[i];
    }
    PoolBuild b;
    const size_t sub_n = (size_t)P * d.K * 3;
    if (int rc = pool_alloc(b, (size_t)P, (size_t)d.K)) return rc;
    UAVRL_CUDA(cudaMemcpy(b.start, start, (size_t)P * 3 * sizeof(double), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(b.goal, goal, (size_t)P * 3 * sizeof(double), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(b.v0, v0.data(), (size_t)P * 3 * sizeof(double), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(b.sub, sub, sub_n * sizeof(double), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(b.nsub, n_sub, (size_t)P * sizeof(int32_t), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(b.alias, al.data(), (size_t)P, cudaMemcpyHostToDevice));
    return pool_install(env, b, P);
}

int uavrl_env_reset(uavrl_env *env, int32_t first, void *stream)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    if (!env->pool_set) return fail(UAVRL_ERR_STATE, "uavrl_env_reset before uavrl_env_set_pool");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    return launch_env_reset(env, first, env->d.n, (cudaStream_t)stream);
}

int uavrl_env_set_reset_stride(uavrl_env *env, int32_t stride)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    if (stride < 1) return fail(UAVRL_ERR_INVALID, "uavrl_env_set_reset_stride: stride must be >= 1");
    env->d.reset_stride = stride;
    return 0;
}

int uavrl_env_observe(uavrl_env *env, float *obs_dev, void *stream)
{
    if (!env || !obs_dev) return fail(UAVRL_ERR_INVALID, "null argument");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_env_observe before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    return launch_env_observe(env, obs_dev, (cudaStream_t)stream);
}

int uavrl_env_step(uavrl_env *env, int32_t action_kind, const void *actions_dev, float *next_obs_dev,
                   float *reward_dev, uint8_t *done_dev, uint8_t *info_dev, uint8_t *collision_dev,
                   uint8_t *ended_dev, void *stream)
{
    if (!env || !actions_dev) return fail(UAVRL_ERR_INVALID, "null argument");
    if (action_kind < 0 || action_kind > 3) return fail(UAVRL_ERR_INVALID, "unknown action_kind");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_env_step before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    return launch_env_step(env, action_kind, actions_dev, next_obs_dev, reward_dev, done_dev, info_dev,
                           collision_dev, ended_dev, (cudaStream_t)stream);
}

int uavrl_env_step_host(uavrl_env *env, int32_t action_kind, const void *actions_host, float *obs_host,
                        float *reward_host, uint8_t *done_host, uint8_t *info_host, uint8_t *coll_host,
                        uint8_t *ended_host)
{
    if (!env || !actions_host) return fail(UAVRL_ERR_INVALID, "null argument");
    if (action_kind < 0 || action_kind > 3) return fail(UAVRL_ERR_INVALID, "unknown action_kind");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_env_step_host before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    const size_t n = (size_t)env->d.n;
    cudaStream_t st = env->own_stream;
    if (int rc = grow(env->staging_mem, env->staging_n, env->d.n, st, false, buf(env->h_act_dev, n), buf(env->h_obs_dev, n * kObsDim),
                      buf(env->h_rew_dev, n), buf(env->h_flags_dev, n * 4)))
        return rc;
    const size_t asz = (action_kind == UAVRL_ACT_CONT_F64 || action_kind == UAVRL_ACT_CONT_F32X2) ? 8 : 4;
    UAVRL_CUDA(cudaMemcpyAsync(env->h_act_dev, actions_host, n * asz, cudaMemcpyHostToDevice, st));
    uint8_t *f = env->h_flags_dev;
    int rc = launch_env_step(env, action_kind, env->h_act_dev, obs_host ? env->h_obs_dev : nullptr,
                             env->h_rew_dev, f, f + n, f + 2 * n, f + 3 * n, st);
    if (rc) return rc;
    if (obs_host) UAVRL_CUDA(cudaMemcpyAsync(obs_host, env->h_obs_dev, n * kObsDim * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (reward_host) UAVRL_CUDA(cudaMemcpyAsync(reward_host, env->h_rew_dev, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (done_host) UAVRL_CUDA(cudaMemcpyAsync(done_host, f, n, cudaMemcpyDeviceToHost, st));
    if (info_host) UAVRL_CUDA(cudaMemcpyAsync(info_host, f + n, n, cudaMemcpyDeviceToHost, st));
    if (coll_host) UAVRL_CUDA(cudaMemcpyAsync(coll_host, f + 2 * n, n, cudaMemcpyDeviceToHost, st));
    if (ended_host) UAVRL_CUDA(cudaMemcpyAsync(ended_host, f + 3 * n, n, cudaMemcpyDeviceToHost, st));
    UAVRL_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int uavrl_env_get_state(uavrl_env *env, const uavrl_env_state_host *o)
{
    if (!env || !o) return fail(UAVRL_ERR_INVALID, "null argument");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const EnvDev &d = env->d;
    const size_t n = (size_t)d.n;
    struct { void *dst; const void *src; size_t sz; } cp[] = {
        { o->px, d.px, 8 }, { o->py, d.py, 8 }, { o->pz, d.pz, 8 }, { o->vx, d.vx, 8 }, { o->vy, d.vy, 8 },
        { o->V, d.V, 8 }, { o->score, d.score, 8 }, { o->total_score, d.total, 8 },
        { o->path_len, d.path_len, 8 }, { o->reward64, d.rew64, 8 }, { o->step, d.step, 4 },
        { o->cursor, d.cursor, 4 }, { o->scenario, d.scen, 4 }, { o->done, d.done, 1 } };
    for (auto &c : cp)
        if (c.dst) UAVRL_CUDA(cudaMemcpy(c.dst, c.src, n * c.sz, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_set_state(uavrl_env *env, const uavrl_env_state_host *in)
{
    if (!env || !in) return fail(UAVRL_ERR_INVALID, "null argument");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_env_set_state before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const EnvDev &d = env->d;
    const size_t n = (size_t)d.n;
    if (in->cursor || in->scenario)
        return fail(UAVRL_ERR_INVALID, "cursor / scenario are owned by the scenario pool: set them through uavrl_env_set_pool + uavrl_env_reset");
    struct { const void *src; void *dst; size_t sz; } cp[] = {
        { in->px, d.px, 8 }, { in->py, d.py, 8 }, { in->pz, d.pz, 8 }, { in->vx, d.vx, 8 }, { in->vy, d.vy, 8 },
        { in->V, d.V, 8 }, { in->score, d.score, 8 }, { in->total_score, d.total, 8 },
        { in->path_len, d.path_len, 8 }, { in->step, d.step, 4 }, { in->done, d.done, 1 } };
    for (auto &c : cp)
        if (c.src) UAVRL_CUDA(cudaMemcpy(c.dst, c.src, n * c.sz, cudaMemcpyHostToDevice));
    env_theta_kernel<<<(d.n + 127) / 128, 128>>>(d);            // the cached heading follows V_vector
    UAVRL_LAUNCHED();
    UAVRL_CUDA(cudaDeviceSynchronize());
    return 0;
}

int uavrl_env_set_extras(uavrl_env *env, const uavrl_env_extras *x)
{
    if (!env || !x) return fail(UAVRL_ERR_INVALID, "null argument");
    if (x->apf_enabled && !x->obstacle_v_host && env->cfg.n_buildings > 0) return fail(UAVRL_ERR_INVALID, "apf_enabled needs obstacle_v_host");
    if (x->track_envs < 0 || x->track_envs > env->d.n || (x->track_envs > 0 && x->track_capacity <= 0))
        return fail(UAVRL_ERR_INVALID, "track_envs must be in [0, n_envs] with a positive track_capacity");
    if (x->energy_enabled && (!(x->v_0 > 0) || !(x->F_b > 0))) return fail(UAVRL_ERR_INVALID, "energy model: v_0 and F_b must be > 0");
    const size_t nv = (size_t)env->cfg.n_buildings * 3;
    // APF and motion read the same attribute of each obstacle (threaten.v): they must agree while both are on
    if (x->apf_enabled && env->motion.on && nv > 0 && memcmp(x->obstacle_v_host, env->motion.v.data(), nv * sizeof(double)) != 0)
        return fail(UAVRL_ERR_INVALID, "apf obstacle_v differs from the velocities of uavrl_env_set_motion");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    // the new extras are built beside the old ones and replace them only once complete
    EnvDev d = env->d;
    DevMem m;
    d.energy = nullptr; d.apf_obs = nullptr; d.sub_env = nullptr; d.path_buf = nullptr; d.path_n = nullptr; d.path_cur = nullptr;
    d.extras = env->d.extras & (kExtraRecord | kExtraMotion); d.track_n = 0; d.track_cap = 0;   // records and motion stay as they are
    const size_t n = (size_t)d.n;
    int rc;
    if (x->energy_enabled) {
        d.pw.P_i = x->P_i; d.pw.v_0 = x->v_0; d.pw.d_0 = x->d_0; d.pw.rho = x->rho; d.pw.s = x->s; d.pw.A = x->A;
        d.pw.P_b = x->P_b; d.pw.F_b = x->F_b; d.pw.xi = x->xi;
        if ((rc = m.alloc(d.energy, n))) return rc;
        d.extras |= kExtraEnergy;
    }
    if (x->apf_enabled) {
        // the obstacle table with velocities; |v| and the direction of v are per-obstacle constants (UAV.py:189,193):
        // Eu_Loc_distance(0, v) and calculate_angle(0, v), evaluated here with libm like the reference does
        std::vector<Cyl> cyl((size_t)(d.k.n_cyl > 0 ? d.k.n_cyl : 1));
        UAVRL_CUDA(cudaMemcpy(cyl.data(), d.cyl, cyl.size() * sizeof(Cyl), cudaMemcpyDeviceToHost));
        std::vector<ApfObs> ob(cyl.size());
        for (int i = 0; i < d.k.n_cyl; ++i) {
            ApfObs o;
            o.x = cyl[i].cx; o.y = cyl[i].cy; o.z = env->base_z.empty() ? 0.0 : env->base_z[(size_t)i]; o.R = cyl[i].R;
            o.vx = x->obstacle_v_host[3 * i]; o.vy = x->obstacle_v_host[3 * i + 1]; o.vz = x->obstacle_v_host[3 * i + 2];
            o.vmag = sqrt(o.vx * o.vx + o.vy * o.vy + o.vz * o.vz);
            const double a = angle_xy(o.vx, o.vy);
            o.cav = cos(a); o.sav = sin(a);
            ob[(size_t)i] = o;
        }
        ApfObs *dob = nullptr;
        if ((rc = m.alloc(dob, ob.size(), false))) return rc;
        UAVRL_CUDA(cudaMemcpy(dob, ob.data(), ob.size() * sizeof(ApfObs), cudaMemcpyHostToDevice));
        d.apf_obs = dob;
        if ((rc = m.alloc(d.sub_env, n * (size_t)d.K * 3))) return rc;
        d.extras |= kExtraApf;
    }
    if (x->track_envs > 0) {
        d.track_n = x->track_envs; d.track_cap = x->track_capacity;
        if ((rc = m.alloc(d.path_buf, (size_t)2 * d.track_n * d.track_cap * 3)) || (rc = m.alloc(d.path_n, (size_t)2 * d.track_n)) ||
            (rc = m.alloc(d.path_cur, (size_t)d.track_n)))
            return rc;
        d.extras |= kExtraTrack;
    }
    UAVRL_CUDA(cudaDeviceSynchronize());                         // nothing may still read the extras being replaced
    env->extras_mem = std::move(m);
    env->d = d;
    if (x->apf_enabled) env->apf_v.assign(x->obstacle_v_host, x->obstacle_v_host + nv);
    else env->apf_v.clear();
    env->extras_set = true;
    env->reset_done = false;                                     // the new columns are initialised by uavrl_env_reset
    return 0;
}

int uavrl_env_get_energy(uavrl_env *env, double *energy_host)
{
    if (!env || !energy_host) return fail(UAVRL_ERR_INVALID, "null argument");
    if (!(env->d.extras & kExtraEnergy)) return fail(UAVRL_ERR_STATE, "the energy model is not enabled (uavrl_env_set_extras)");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(energy_host, env->d.energy, (size_t)env->d.n * 8, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_get_energy_total(uavrl_env *env, double *total_out)
{
    if (!env || !total_out) return fail(UAVRL_ERR_INVALID, "null argument");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(total_out, env->d.stat_reward + 1, 8, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_get_path(uavrl_env *env, int32_t e, int32_t which, int32_t capacity, double *xyz_host, int32_t *n_out)
{
    if (!env || !xyz_host || !n_out || capacity <= 0 || which < 0 || which > 1) return fail(UAVRL_ERR_INVALID, "bad argument");
    const EnvDev &d = env->d;
    if (!(d.extras & kExtraTrack) || e < 0 || e >= d.track_n) return fail(UAVRL_ERR_STATE, "this UAV is not tracked (uavrl_env_set_extras track_envs)");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    int32_t cur = 0, np = 0;
    UAVRL_CUDA(cudaMemcpy(&cur, d.path_cur + e, 4, cudaMemcpyDeviceToHost));
    const int buf = which == 0 ? cur : (cur ^ 1);
    UAVRL_CUDA(cudaMemcpy(&np, d.path_n + (size_t)buf * d.track_n + e, 4, cudaMemcpyDeviceToHost));
    *n_out = np;
    int m = np < d.track_cap ? np : d.track_cap;
    if (m > capacity) m = capacity;
    if (m > 0) UAVRL_CUDA(cudaMemcpy(xyz_host, d.path_buf + ((size_t)buf * d.track_n + e) * d.track_cap * 3, (size_t)m * 24, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_get_subgoals(uavrl_env *env, double *sub_host)
{
    if (!env || !sub_host) return fail(UAVRL_ERR_INVALID, "null argument");
    const EnvDev &d = env->d;
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_env_get_subgoals before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const size_t row = (size_t)d.K * 3;
    if (d.extras & kExtraApf) {
        UAVRL_CUDA(cudaMemcpy(sub_host, d.sub_env, (size_t)d.n * row * 8, cudaMemcpyDeviceToHost));
        return 0;
    }
    std::vector<int32_t> scen((size_t)d.n);
    UAVRL_CUDA(cudaMemcpy(scen.data(), d.scen, (size_t)d.n * 4, cudaMemcpyDeviceToHost));
    for (int e = 0; e < d.n; ++e)
        UAVRL_CUDA(cudaMemcpy(sub_host + (size_t)e * row, d.pool_sub + (size_t)scen[(size_t)e] * row, row * 8, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_set_records(uavrl_env *env, int64_t capacity)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    if (capacity < 0) return fail(UAVRL_ERR_INVALID, "uavrl_env_set_records: capacity must be >= 0");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    EnvRecords r;                                                // built beside the old records, swapped in once complete
    if (capacity > 0)
        if (int rc = records_alloc(r, env->d.n, capacity)) return rc;
    UAVRL_CUDA(cudaDeviceSynchronize());                         // nothing may still write the records being replaced
    env->records = std::move(r);
    env->d.extras = capacity > 0 ? (env->d.extras | kExtraRecord) : (env->d.extras & ~kExtraRecord);
    return 0;
}

int uavrl_env_get_records(uavrl_env *env, int64_t capacity, uavrl_episode_record *records_host, int64_t *n_written_out,
                          int64_t *n_dropped_out, int32_t clear)
{
    if (!env || capacity < 0 || (capacity > 0 && !records_host)) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (!env->records.on) return fail(UAVRL_ERR_STATE, "episode records are not enabled (uavrl_env_set_records)");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const EnvRecDev &r = env->records.dev;
    const int64_t m = capacity < r.cap ? capacity : r.cap;
    if (m > 0) UAVRL_CUDA(cudaMemcpy(records_host, r.rec, (size_t)m * sizeof(uavrl_episode_record), cudaMemcpyDeviceToHost));
    unsigned long long c[2];
    UAVRL_CUDA(cudaMemcpy(c, r.counts, sizeof(c), cudaMemcpyDeviceToHost));
    if (n_written_out) *n_written_out = (int64_t)c[0];
    if (n_dropped_out) *n_dropped_out = (int64_t)c[1];
    if (clear) {
        if (int rc = records_clear(env->records, env->d.n, nullptr)) return rc;
        UAVRL_CUDA(cudaDeviceSynchronize());
    }
    return 0;
}

int uavrl_env_clear_records(uavrl_env *env)
{
    return uavrl_env_get_records(env, 0, nullptr, nullptr, nullptr, 1);
}

int uavrl_env_threaten_rate(uavrl_env *env, int32_t n, const double *pts_host, uint8_t *out_host)
{
    if (!env || n <= 0 || !pts_host || !out_host) return fail(UAVRL_ERR_INVALID, "null/empty argument");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    DevMem m;
    double *dp = nullptr; uint8_t *dout = nullptr;
    int rc;
    if ((rc = m.alloc(dp, (size_t)n * 3, false)) || (rc = m.alloc(dout, (size_t)n, false))) return rc;
    UAVRL_CUDA(cudaMemcpy(dp, pts_host, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice));
    threat_kernel<<<(n + 127) / 128, 128>>>(env->d, n, dp, dout, env->motion.on ? env->motion.buf[env->motion.cur] : nullptr);
    UAVRL_LAUNCHED();
    UAVRL_CUDA(cudaMemcpy(out_host, dout, (size_t)n, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_env_set_motion(uavrl_env *env, const double *position_host, const double *velocity_host)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    const int nc = env->cfg.n_buildings;
    const double len = env->cfg.len, width = env->cfg.width;
    if (!velocity_host && position_host)
        return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: positions without velocities (motion off keeps the cylinders as created)");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    if (!velocity_host) {                                        // motion off: the step reads the cylinders as created again
        UAVRL_CUDA(cudaDeviceSynchronize());
        env->motion = EnvMotion();
        env->d.extras &= ~kExtraMotion;
        return 0;
    }
    if (nc == 0) return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: the city has no obstacles");
    // the centres: the ones given, or the current ones (the moving table, else the cylinders as created)
    std::vector<MoveObs> rows((size_t)nc);
    if (position_host) {
        for (int i = 0; i < nc; ++i) { rows[(size_t)i].x = position_host[3 * i]; rows[(size_t)i].y = position_host[3 * i + 1]; }
    } else {
        UAVRL_CUDA(cudaDeviceSynchronize());
        if (env->motion.on) {
            UAVRL_CUDA(cudaMemcpy(rows.data(), env->motion.buf[env->motion.cur], (size_t)nc * sizeof(MoveObs), cudaMemcpyDeviceToHost));
        } else {
            std::vector<Cyl> cyl((size_t)nc);
            UAVRL_CUDA(cudaMemcpy(cyl.data(), env->d.cyl, (size_t)nc * sizeof(Cyl), cudaMemcpyDeviceToHost));
            for (int i = 0; i < nc; ++i) { rows[(size_t)i].x = cyl[(size_t)i].cx; rows[(size_t)i].y = cyl[(size_t)i].cy; }
        }
    }
    double vmax = 0.0;
    for (int i = 0; i < nc; ++i) {
        MoveObs &o = rows[(size_t)i];
        o.vx = velocity_host[3 * i]; o.vy = velocity_host[3 * i + 1];
        const double vz = velocity_host[3 * i + 2];
        if (!std::isfinite(o.x) || !std::isfinite(o.y) || !std::isfinite(o.vx) || !std::isfinite(o.vy) || !std::isfinite(vz))
            return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: non-finite position or velocity");
        if (o.x < 0.0 || o.x > len || o.y < 0.0 || o.y > width)
            return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: a centre lies outside [0, len] x [0, width]");
        if (fabs(o.vx) > len || fabs(o.vy) > width)
            return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: |vx| must be <= len and |vy| <= width");
        vmax = fmax(vmax, fmax(fabs(o.vx), fabs(o.vy)));
    }
    const size_t nv = (size_t)nc * 3;
    if ((env->d.extras & kExtraApf) && memcmp(velocity_host, env->apf_v.data(), nv * sizeof(double)) != 0)
        return fail(UAVRL_ERR_INVALID, "uavrl_env_set_motion: velocities differ from the APF model's obstacle_v");
    // cos / sin of calculate_angle(0, v) for the four sign variants, with libm like uavrl_env_set_extras
    std::vector<double> dir((size_t)nc * 8);
    for (int i = 0; i < nc; ++i)
        for (int v = 0; v < 4; ++v) {
            const MoveObs &o = rows[(size_t)i];
            const double a = angle_xy(copysign(o.vx, (v & 1) ? -1.0 : 1.0), copysign(o.vy, (v & 2) ? -1.0 : 1.0));
            dir[(size_t)i * 8 + 2 * v] = cos(a); dir[(size_t)i * 8 + 2 * v + 1] = sin(a);
        }
    EnvMotion mo;                                                // built beside the old table, swapped in once complete
    int rc;
    if ((rc = mo.mem.alloc(mo.buf[0], (size_t)nc, false)) || (rc = mo.mem.alloc(mo.buf[1], (size_t)nc, false)) ||
        (rc = mo.mem.alloc(mo.dir, dir.size(), false)))
        return rc;
    UAVRL_CUDA(cudaMemcpy(mo.buf[0], rows.data(), (size_t)nc * sizeof(MoveObs), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(mo.buf[1], rows.data(), (size_t)nc * sizeof(MoveObs), cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(mo.dir, dir.data(), dir.size() * sizeof(double), cudaMemcpyHostToDevice));
    mo.v.assign(velocity_host, velocity_host + nv);
    mo.reach = vmax + 1.0;                                       // a metre of margin over the rounded centre moves
    mo.on = true;
    UAVRL_CUDA(cudaDeviceSynchronize());                         // nothing may still read the table being replaced
    env->motion = std::move(mo);
    env->d.extras |= kExtraMotion;
    return 0;
}

int uavrl_env_get_obstacles(uavrl_env *env, double *position_host, double *velocity_host, int64_t *steps_out)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    const int nc = env->cfg.n_buildings;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const EnvMotion &mo = env->motion;
    std::vector<MoveObs> rows((size_t)(nc > 0 ? nc : 1));
    if (mo.on) {
        UAVRL_CUDA(cudaMemcpy(rows.data(), mo.buf[mo.cur], (size_t)nc * sizeof(MoveObs), cudaMemcpyDeviceToHost));
    } else if (nc > 0) {
        std::vector<Cyl> cyl((size_t)nc);
        UAVRL_CUDA(cudaMemcpy(cyl.data(), env->d.cyl, (size_t)nc * sizeof(Cyl), cudaMemcpyDeviceToHost));
        for (int i = 0; i < nc; ++i) rows[(size_t)i] = MoveObs{ cyl[(size_t)i].cx, cyl[(size_t)i].cy, 0.0, 0.0 };
    }
    for (int i = 0; i < nc; ++i) {
        const MoveObs &o = rows[(size_t)i];
        if (position_host) { position_host[3 * i] = o.x; position_host[3 * i + 1] = o.y; position_host[3 * i + 2] = env->base_z[(size_t)i]; }
        if (velocity_host) {
            velocity_host[3 * i] = o.vx; velocity_host[3 * i + 1] = o.vy;
            velocity_host[3 * i + 2] = mo.on ? mo.v[(size_t)i * 3 + 2] : 0.0;
        }
    }
    if (steps_out) *steps_out = mo.on ? mo.steps : 0;
    return 0;
}

}  // extern "C"
