// scenario.cu -- scenario generator: UAV.reset() draws + RRT sub-goal queues (arithmetic in rrt_core.cuh).
//
//   uavrl_make_scenarios      host threads, host arrays out (feeds uavrl_env_set_pool)
//   uavrl_env_generate_pool   device kernel, one warp per scenario (tree in shared memory), writes the env's device pool directly
//                             (SURVEY.md 8f-1: with tens of thousands of auto-resetting envs the host RRT is the
//                             bottleneck); bit-identical to the host generator for the same (seed, index)
//   uavrl_env_get_pool        read a device pool back (tests, checkpoints)
#include <math.h>

#include <atomic>
#include <thread>
#include <vector>

#include "common.cuh"
#include "env.cuh"
#include "rrt_core.cuh"

namespace uavrl {
namespace {

void fill_city(const uavrl_env_config *cfg, RrtCity &c, std::vector<Cyl> &cyl)
{
    c.k.width = cfg->width; c.k.h = cfg->h; c.k.max_v = cfg->max_v; c.k.min_v = cfg->min_v;
    c.k.steering = cfg->steering_angle; c.k.climb = cfg->climb_rate; c.k.max_step = cfg->max_step;
    c.k.n_cyl = cfg->n_buildings; c.len = cfg->len;
    for (int i = 0; i < cfg->n_buildings; ++i) {
        const double *b = cfg->buildings_host + 5 * i;
        Cyl cy; cy.cx = b[0]; cy.cy = b[1]; cy.R = b[3]; cy.H = b[4];
        const double r2 = cy.R * cy.R; cy.r2lo = r2 * (1.0 - 1e-12); cy.r2hi = r2 * (1.0 + 1e-12);
        cyl.push_back(cy);
    }
    c.cyl = cyl.data();
}

// ---- device generator: one WARP per scenario, tree in shared memory (SoA) -------------------------------------------
// Same arithmetic and the same decisions as rrt_core.cuh's sequential rrt_plan (the test compares the pools bit for
// bit): every lane runs the counter-based RNG redundantly, the nearest-node search and the parent choice are strided
// over the lanes and reduced with "smallest value, then smallest index" (= the sequential first minimum), the 5 m
// collision samples of one edge are spread over the lanes.
constexpr int kRrtWarpsPerCta = 2;

struct WarpTree {
    double x[kRrtMaxNodes], y[kRrtMaxNodes], z[kRrtMaxNodes], cost[kRrtMaxNodes];
    int32_t parent[kRrtMaxNodes];
};

__device__ __forceinline__ void warp_argmin(double &v, int &i)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
}

// RRT.py:48-56 with the sample points spread over the lanes (<= 32 points: an edge is at most one RRT step long)
__device__ __forceinline__ bool warp_obstacle_free(const RrtCity &c, double ax, double ay, double az, double bx, double by, double bz,
                                                   double step_size, int lane)
{
    const int steps = (int)ddiv(dist3(ax, ay, az, bx, by, bz), step_size);
    const double den = (double)(steps + 1);
    const double dx = dsub(bx, ax), dy = dsub(by, ay), dz = dsub(bz, az);
    bool hit = false;
    for (int i = lane; i <= steps; i += 32) {
        const double fi = (double)i;
        hit |= rrt_threat(c, dadd(ax, ddiv(dmul(dx, fi), den)), dadd(ay, ddiv(dmul(dy, fi), den)), dadd(az, ddiv(dmul(dz, fi), den))) == 1;
    }
    return __ballot_sync(0xffffffffu, hit) == 0u;
}

__device__ int rrt_plan_warp(const RrtCity &c, RrtRng &rng, const P3 &start, const P3 &goal, double step_size, WarpTree &tr, double *path,
                             int K, int lane)
{
    const double obstacle_step = 5.0;
    int n = 1, goal_parent = -1;
    if (lane == 0) { tr.x[0] = start.x; tr.y[0] = start.y; tr.z[0] = start.z; tr.cost[0] = 0.0; tr.parent[0] = -1; }
    __syncwarp();
    for (int it = 0; it < kRrtMaxIter; ++it) {
        double rx, ry, rz;
        if (rng.uniform(0.0, 1.0) > 0.5) {
            rx = rng.uniform(0.0, c.len); ry = rng.uniform(0.0, c.k.width); rz = rng.uniform(0.0, c.k.h);
        } else {
            rx = goal.x; ry = goal.y; rz = goal.z;
        }
        double best = 1e300; int nearest = 0x7fffffff;
        for (int i = lane; i < n; i += 32) {
            const double dd = dist3(tr.x[i], tr.y[i], tr.z[i], rx, ry, rz);
            if (dd < best) { best = dd; nearest = i; }
        }
        warp_argmin(best, nearest);
        const double fx = tr.x[nearest], fy = tr.y[nearest], fz = tr.z[nearest];
        const double dx = dsub(rx, fx), dy = dsub(ry, fy), dz = dsub(rz, fz);
        const double length = dsqrt(dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz)));
        double nx, ny, nz;
        if (length < step_size) { nx = rx; ny = ry; nz = rz; }
        else {
            nx = dadd(fx, dmul(ddiv(dx, length), step_size));
            ny = dadd(fy, dmul(ddiv(dy, length), step_size));
            nz = dadd(fz, dmul(ddiv(dz, length), step_size));
        }
        if (!warp_obstacle_free(c, fx, fy, fz, nx, ny, nz, obstacle_step, lane)) continue;
        if (n >= kRrtMaxNodes) return 0;
        const int me = n++;
        const double cost0 = dadd(tr.cost[nearest], dist3(fx, fy, fz, nx, ny, nz));
        // cheaper parent among the nodes within one step: min (cost_i + d_i) over collision-free candidates below cost0,
        // first index on ties == the sequential scan with its running minimum (RRT.py:86-92)
        double bc = cost0; int bp = 0x7fffffff;
        for (int i = lane; i < me; i += 32) {
            const double dd = dist3(tr.x[i], tr.y[i], tr.z[i], nx, ny, nz);
            const double ci = dadd(tr.cost[i], dd);
            if (dd < step_size && bc > ci) {
                if (rrt_obstacle_free(c, tr.x[i], tr.y[i], tr.z[i], nx, ny, nz, obstacle_step)) { bc = ci; bp = i; }
            }
        }
        warp_argmin(bc, bp);
        __syncwarp();
        if (lane == 0) {
            tr.x[me] = nx; tr.y[me] = ny; tr.z[me] = nz;
            tr.parent[me] = (bp != 0x7fffffff) ? bp : nearest;
            tr.cost[me] = (bp != 0x7fffffff) ? bc : cost0;
        }
        __syncwarp();
        if (dist3(nx, ny, nz, goal.x, goal.y, goal.z) <= step_size) { goal_parent = me; break; }
    }
    if (goal_parent < 0) return 0;
    int len = 1;
    for (int i = goal_parent; i >= 0; i = tr.parent[i]) ++len;
    if (len > K) return 0;
    if (lane == 0) {
        int w = len - 1;
        path[3 * w] = goal.x; path[3 * w + 1] = goal.y; path[3 * w + 2] = goal.z;
        for (int i = goal_parent; i >= 0; i = tr.parent[i]) { --w; path[3 * w] = tr.x[i]; path[3 * w + 1] = tr.y[i]; path[3 * w + 2] = tr.z[i]; }
    }
    __syncwarp();
    return len;
}

__global__ void __launch_bounds__(32 * kRrtWarpsPerCta)
rrt_pool_kernel(RrtCity c, uint64_t seed, int P, double step, int K, double *start, double *goal, double *v0, double *sub,
                int32_t *n_sub, uint8_t *alias, int *failed)
{
    extern __shared__ __align__(16) unsigned char rrt_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.x * kRrtWarpsPerCta + warp;
    if (s >= P) return;
    WarpTree &tr = reinterpret_cast<WarpTree *>(rrt_smem)[warp];
    double *q = sub + (size_t)s * K * 3;
    int len = 0;
    double seta = 0.0;
    P3 st, gl;
    for (int attempt = 0; attempt < kRrtAttempts && len == 0; ++attempt) {           // make_scenario (rrt_core.cuh), per warp
        RrtRng rng;
        rng.init(seed, ((uint64_t)s << 8) | (uint64_t)attempt);
        seta = rng.uniform(0.0, 2 * kPi);
        st.x = rng.uniform(10.0, 210.0); st.y = rng.uniform(1.0, 10.0); st.z = 0.0;
        gl.x = rng.uniform(330.0, 490.0); gl.y = rng.uniform(420.0, 490.0); gl.z = 0.0;
        len = rrt_plan_warp(c, rng, st, gl, step, tr, q, K, lane);
    }
    if (len == 0) { if (lane == 0) { atomicExch(failed, 1); n_sub[s] = 0; } return; }
    for (int i = 3 * len + lane; i < 3 * K; i += 32) q[i] = 0.0;
    if (lane == 0) {
        n_sub[s] = len;
        alias[s] = 1;                                   // RRT.py:69: queue[0] is the UAV's own position object
        start[3 * (size_t)s] = st.x; start[3 * (size_t)s + 1] = st.y; start[3 * (size_t)s + 2] = st.z;
        goal[3 * (size_t)s] = gl.x; goal[3 * (size_t)s + 1] = gl.y; goal[3 * (size_t)s + 2] = gl.z;
        // UAV.py:344-348: V_vector = Max_V*(cos, sin)(heading); V = Calc_V()
        double vx = dmul(c.k.max_v, cos(seta)), vy = dmul(c.k.max_v, sin(seta));
        const double V = calc_v(c.k, vx, vy);
        v0[3 * (size_t)s] = vx; v0[3 * (size_t)s + 1] = vy; v0[3 * (size_t)s + 2] = V;
    }
}

}  // namespace
}  // namespace uavrl

using namespace uavrl;

extern "C" int uavrl_make_scenarios(const uavrl_env_config *cfg, uint64_t seed, int32_t P, int32_t rrt_step,
                                    double *start, double *goal, double *heading, double *sub, int32_t *n_sub)
{
    if (!cfg || P <= 0 || !start || !goal || !heading || !sub || !n_sub)
        return fail(UAVRL_ERR_INVALID, "uavrl_make_scenarios: null/empty argument");
    if (cfg->n_buildings > 0 && !cfg->buildings_host) return fail(UAVRL_ERR_INVALID, "buildings_host is null");
    RrtCity c;
    std::vector<Cyl> cyl;
    fill_city(cfg, c, cyl);
    const int K = cfg->max_subgoals;
    const double step = rrt_step > 0 ? (double)rrt_step : 30.0;       // config/UAV.xml sub_granularity
    // scenarios are independent: spread them over the host cores
    unsigned nthreads = std::thread::hardware_concurrency();
    if (nthreads == 0) nthreads = 1;
    if (nthreads > 64) nthreads = 64;
    if ((int)nthreads > P) nthreads = (unsigned)P;
    std::atomic<int> next{0}, failed{0};
    auto worker = [&]() {
        std::vector<RrtNode> nodes(kRrtMaxNodes);
        for (int s = next.fetch_add(1); s < P; s = next.fetch_add(1)) {
            n_sub[s] = make_scenario(c, seed, s, step, K, nodes.data(), start + 3 * (size_t)s, goal + 3 * (size_t)s,
                                     heading + s, sub + (size_t)s * K * 3);
            if (n_sub[s] == 0) failed.store(1);
        }
    };
    std::vector<std::thread> pool;
    for (unsigned i = 0; i < nthreads; ++i) pool.emplace_back(worker);
    for (auto &th : pool) th.join();
    if (failed.load()) return fail(UAVRL_ERR_INVALID, "RRT found no path within max_subgoals for a scenario");
    return 0;
}

extern "C" int uavrl_env_generate_pool(uavrl_env *env, int32_t P, uint64_t seed, int32_t rrt_step, void *stream)
{
    if (!env || P <= 0) return fail(UAVRL_ERR_INVALID, "uavrl_env_generate_pool: null/empty argument");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    EnvDev &d = env->d;
    cudaStream_t st = (cudaStream_t)stream;
    RrtCity c;
    c.k = d.k; c.len = env->cfg.len; c.cyl = d.cyl;
    const double step = rrt_step > 0 ? (double)rrt_step : 30.0;
    PoolBuild b;
    DevMem tmp;
    int *failed = nullptr;
    int rc;
    if ((rc = pool_alloc(b, (size_t)P, (size_t)d.K)) || (rc = tmp.alloc(failed, 1, false))) return rc;
    UAVRL_CUDA(cudaMemsetAsync(failed, 0, sizeof(int), st));
    const size_t smem = sizeof(WarpTree) * kRrtWarpsPerCta;          // 2 x 18 KB
    UAVRL_CUDA(cudaFuncSetAttribute(rrt_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // per device: set on every call
    const int blocks = (P + kRrtWarpsPerCta - 1) / kRrtWarpsPerCta;
    rrt_pool_kernel<<<blocks, 32 * kRrtWarpsPerCta, smem, st>>>(c, seed, P, step, d.K, b.start, b.goal, b.v0, b.sub, b.nsub, b.alias,
                                                                 failed);
    UAVRL_LAUNCHED();
    int h_failed = 0;
    UAVRL_CUDA(cudaMemcpyAsync(&h_failed, failed, sizeof(int), cudaMemcpyDeviceToHost, st));
    UAVRL_CUDA(cudaStreamSynchronize(st));
    if (h_failed) return fail(UAVRL_ERR_INVALID, "device RRT found no path within max_subgoals for a scenario");
    return pool_install(env, b, P);
}

extern "C" int uavrl_env_get_pool(uavrl_env *env, double *start, double *goal, double *v0, double *sub, int32_t *n_sub)
{
    if (!env) return fail(UAVRL_ERR_INVALID, "null env");
    if (!env->pool_set) return fail(UAVRL_ERR_STATE, "uavrl_env_get_pool before a pool was set");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const EnvDev &d = env->d;
    const size_t P = (size_t)d.P;
    if (start) UAVRL_CUDA(cudaMemcpy(start, d.pool_start, P * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (goal) UAVRL_CUDA(cudaMemcpy(goal, d.pool_goal, P * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (v0) UAVRL_CUDA(cudaMemcpy(v0, d.pool_v0, P * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (sub) UAVRL_CUDA(cudaMemcpy(sub, d.pool_sub, P * d.K * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (n_sub) UAVRL_CUDA(cudaMemcpy(n_sub, d.pool_nsub, P * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return 0;
}
