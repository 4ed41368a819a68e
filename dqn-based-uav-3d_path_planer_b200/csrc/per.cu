// per.cu -- prioritised replay kernels and the tree operations of the replay store (design in per.cuh).
#include "per.cuh"

#include <math.h>

#include <vector>

#include "replay.cuh"

namespace uavrl {

__device__ __forceinline__ int64_t per_pos(const PerDev &p, int64_t slot) { int64_t j = slot - p.rot; return j < 0 ? j + p.cap : j; }
__device__ __forceinline__ int64_t per_slot(const PerDev &p, int64_t pos) { int64_t s = pos + p.rot; return s >= p.cap ? s - p.cap : s; }

// fixed-order sum of one value per lane (xor butterfly: every lane ends with the same bits)
__device__ __forceinline__ double warp_sum(double x)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}
__device__ __forceinline__ double warp_scan_incl(double x, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const double y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    return x;
}

// ---- leaves
// mode 0: explicit priorities; 1: ReplayTree.push (:152-154)  p = (|e| + eps)^alpha ; 2: batch_update (:216-221) with the clip.
// The reference computes both in float32 (the errors arrive as float32 tensors / arrays).
// Trainer blockIdx.y: its tree, and row g of [G][n] slots / priorities / errors (a range fill covers the same slots of every tree).
__global__ void per_leaf_kernel(PerDev p, int n, const int32_t *__restrict__ slots, int64_t first, const double *__restrict__ prio,
                                const float *__restrict__ err, int mode, double fill, int n_first, double fill_rest)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t r = (size_t)blockIdx.y * (size_t)n + (size_t)i;
    const int64_t s = slots ? (int64_t)slots[r] : (first + i) % p.cap;
    double v;
    if (mode == 0) v = prio ? prio[r] : (i < n_first ? fill : fill_rest);
    else {
        float e = fabsf(err[r]) + (float)p.eps;
        if (mode == 2) e = fminf(e, (float)p.err_upper);
        v = (double)powf(e, (float)p.alpha);
    }
    p.leaf[(size_t)blockIdx.y * (size_t)p.cap + s] = v;
}

// one warp per touched slot: recompute the l1 entry (level 1) or the l2 entry (level 2) that covers it
__global__ void per_level_kernel(PerDev p, int n, const int32_t *__restrict__ slots, int64_t first, int level)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    const size_t t = blockIdx.y;                                  // trainer: its tree and row t of [G][n] slots
    const double *leaf = p.leaf + t * (size_t)p.cap;
    double *l1 = p.l1 + t * (size_t)p.n1, *l2 = p.l2 + t * (size_t)p.n2;
    const int64_t s = slots ? (int64_t)slots[t * (size_t)n + w] : (first + w) % p.cap;
    const int64_t pos = per_pos(p, s);
    if (level == 1) {
        const int64_t g = pos >> 5, j = (g << 5) + lane;
        const double x = j < p.cap ? leaf[per_slot(p, j)] : 0.0;
        const double sum = warp_sum(x);
        if (lane == 0) l1[g] = sum;
    } else {
        const int64_t b = pos >> 10, j = (b << 5) + lane;
        const double x = j < p.n1 ? l1[j] : 0.0;
        const double sum = warp_sum(x);
        if (lane == 0) l2[b] = sum;
    }
}

// ---- ReplayTree.sample2 (:186-213)
// Trainer blockIdx.y samples B from its own tree with its own key (trainer_key: what a stand-alone learner seeded with seed + g
// draws), into row g of the [G][B] outputs, and normalises by its own maximum weight (wmax_bits[g]).
__global__ void __launch_bounds__(256) per_sample_kernel(PerDev p, int B, const double *__restrict__ u_tape, uint64_t key, uint64_t call,
                                                         double n_entries, double beta, int32_t *__restrict__ slot_out,
                                                         double *__restrict__ w_raw, unsigned long long *wmax_bits)
{
    __shared__ double pre[kPerMaxL2];       // inclusive prefix of l2
    __shared__ double wsum[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t t = blockIdx.y, r0 = t * (size_t)B;
    p.leaf += t * (size_t)p.cap; p.l1 += t * (size_t)p.n1; p.l2 += t * (size_t)p.n2;
    if (u_tape) u_tape += r0;
    slot_out += r0; w_raw += r0; wmax_bits += t;
    key = trainer_key(key, kPerSalt, (int)t);
    // inclusive scan of l2 (n2 <= 4096): 16 consecutive entries per thread, then a scan of the 256 thread totals
    constexpr int PER_T = kPerMaxL2 / 256;
    double loc[PER_T], run = 0.0;
#pragma unroll
    for (int k = 0; k < PER_T; ++k) { const int j = tid * PER_T + k; run += (j < p.n2) ? p.l2[j] : 0.0; loc[k] = run; }
    double incl = warp_scan_incl(run, lane);
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    double off = incl - run;
    for (int wv = 0; wv < warp; ++wv) off += wsum[wv];
#pragma unroll
    for (int k = 0; k < PER_T; ++k) pre[tid * PER_T + k] = off + loc[k];
    __syncthreads();
    const int n2 = (int)p.n2;
    const double total = floor(pre[n2 - 1]);                  // SumTree.total(): int(tree[0])
    const double seg = total / (double)B;                    // :187
    for (int i = blockIdx.x * 8 + warp; i < B; i += gridDim.x * 8) {
        double u;
        if (u_tape) u = u_tape[i];
        else {
            uint32_t r[4];
            Philox::gen(key, call, (uint64_t)i, r);
            u = (double)(((uint64_t)(r[0] >> 5) << 26) | (uint64_t)(r[1] >> 6)) * (1.0 / 9007199254740992.0);
        }
        const double a = seg * (double)i, b = seg * (double)(i + 1);
        const double s = a + (b - a) * u;                     // random.uniform(a, b)   :199-202
        // first l2 entry whose inclusive prefix reaches s  (get_leaf: `v <= tree[left]` goes left)
        int lo = 0, hi = n2 - 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (pre[mid] >= s) hi = mid; else lo = mid + 1; }
        double v = s - (lo > 0 ? pre[lo - 1] : 0.0);
        // level 1: the 32 group sums of that block
        const int64_t g0 = (int64_t)lo << 5;
        double x = (g0 + lane < p.n1) ? p.l1[g0 + lane] : 0.0;
        double ix = warp_scan_incl(x, lane);
        unsigned m = __ballot_sync(0xffffffffu, ix >= v && (g0 + lane < p.n1));
        unsigned valid1 = __ballot_sync(0xffffffffu, g0 + lane < p.n1 && x > 0.0);
        if (!valid1) valid1 = __ballot_sync(0xffffffffu, g0 + lane < p.n1);
        int j1 = m ? __ffs(m) - 1 : 31 - __clz(valid1);
        v -= __shfl_sync(0xffffffffu, ix - x, j1);
        // level 0: the 32 leaves of that group
        const int64_t p0 = (g0 + j1) << 5;
        x = (p0 + lane < p.cap) ? p.leaf[per_slot(p, p0 + lane)] : 0.0;
        ix = warp_scan_incl(x, lane);
        m = __ballot_sync(0xffffffffu, ix >= v && (p0 + lane < p.cap));
        unsigned valid0 = __ballot_sync(0xffffffffu, p0 + lane < p.cap && x > 0.0);     // rounding fall-through: last stored leaf
        if (!valid0) valid0 = __ballot_sync(0xffffffffu, p0 + lane < p.cap);
        const int j0 = m ? __ffs(m) - 1 : 31 - __clz(valid0);
        const double pr = __shfl_sync(0xffffffffu, x, j0);
        if (lane == 0) {
            slot_out[i] = (int32_t)per_slot(p, p0 + j0);
            const double prob = pr / total;                   // :206-208
            const double w = pow(n_entries * prob, -beta);    // :209
            w_raw[i] = w;
            atomicMax(wmax_bits, (unsigned long long)__double_as_longlong(w));      // positive doubles order like their bit patterns
        }
    }
}

__global__ void per_norm_kernel(int B, const double *__restrict__ w_raw, const unsigned long long *wmax_bits, float *__restrict__ w)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t r = (size_t)blockIdx.y * (size_t)B + (size_t)i;  // row blockIdx.y: that trainer's own maximum
    if (i < B) w[r] = (float)(w_raw[r] / __longlong_as_double((long long)wmax_bits[blockIdx.y]));      // :210
}

static int per_refresh(const PerDev &p, int n, const int32_t *slots, int64_t first, cudaStream_t st)
{
    const dim3 blocks((unsigned)(((int64_t)n * 32 + 255) / 256), (unsigned)p.G);
    per_level_kernel<<<blocks, 256, 0, st>>>(p, n, slots, first, 1);
    UAVRL_LAUNCHED();
    per_level_kernel<<<blocks, 256, 0, st>>>(p, n, slots, first, 2);
    UAVRL_LAUNCHED();
    return 0;
}

int ReplayStore::per_enable(double alpha, double beta0, double beta_inc, double eps, double err_upper)
{
    if (per.dev.enabled) return fail(UAVRL_ERR_STATE, "prioritised replay is already enabled");
    if (count != 0) return fail(UAVRL_ERR_STATE, "enable prioritised replay before the first transition is stored");
    if (G > 1 && mode != kReplayLockstep)
        return fail(UAVRL_ERR_INVALID, "prioritised replay on a learner with several trainers needs the lockstep ring (lockstep_envs > 0)");
    PerDev p;                                                     // swapped in once complete
    memset(&p, 0, sizeof(p));
    p.G = G;
    p.cap = slots / G;                                            // trainer-local slots: ring_frames x Ng
    int64_t pow2 = 1;
    while (pow2 < p.cap) pow2 <<= 1;
    p.rot = pow2 - p.cap;
    p.n1 = (p.cap + 31) / 32; p.n2 = (p.n1 + 31) / 32;
    if (p.n2 > kPerMaxL2) return fail(UAVRL_ERR_INVALID, "prioritised replay supports at most 4194304 slots");
    p.alpha = alpha >= 0 ? alpha : 0.6; p.beta = beta0 >= 0 ? beta0 : 0.4; p.beta_inc = beta_inc >= 0 ? beta_inc : 0.001;   // :141-148
    p.eps = eps >= 0 ? eps : 0.01; p.err_upper = err_upper >= 0 ? err_upper : 1.0;
    int rc;
    const size_t Gs = (size_t)p.G;
    DevMem m;
    if ((rc = m.alloc(p.leaf, Gs * p.cap)) || (rc = m.alloc(p.l1, Gs * p.n1)) || (rc = m.alloc(p.l2, Gs * p.n2)) ||
        (rc = m.alloc(p.wmax_bits, Gs)))
        return rc;
    p.enabled = 1;
    per.dev = p;
    per.mem = std::move(m);
    return 0;
}

int ReplayStore::per_fill_range(int64_t first_slot, int64_t n, double value, cudaStream_t st, int64_t n_first, double value_rest)
{
    if (n <= 0) return 0;
    const PerDev &p = per.dev;
    per_leaf_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)p.G), 256, 0, st>>>(p, (int)n, nullptr, first_slot % p.cap, nullptr,
                                                                                   nullptr, 0, value, (int)(n_first < 0 ? n : n_first),
                                                                                   value_rest);
    UAVRL_LAUNCHED();
    return per_refresh(p, (int)n, nullptr, first_slot % p.cap, st);
}

int ReplayStore::per_set(int n, const int32_t *slot_in, const double *prio, const float *abs_err, int clip, cudaStream_t st)
{
    const PerDev &p = per.dev;
    per_leaf_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)p.G), 256, 0, st>>>(p, n, slot_in, 0, prio, abs_err,
                                                                                   prio ? 0 : (clip ? 2 : 1), 0.0, n, 0.0);
    UAVRL_LAUNCHED();
    return per_refresh(p, n, slot_in, 0, st);
}

int ReplayStore::per_sample(uint64_t seed, int B, const double *u_tape, int32_t *slot_out, float *w_out, cudaStream_t st)
{
    PerDev &p = per.dev;
    const size_t Gs = (size_t)p.G;
    if (int rc = grow(per.scratch_mem, p.scratch_cap, B, st, false, buf(p.idx, Gs * B), buf(p.w, Gs * B), buf(p.abs_err, Gs * B),
                      buf(p.w_raw, Gs * B)))
        return rc;
    p.beta = fmin(1.0, p.beta + p.beta_inc);                  // :195
    UAVRL_CUDA(cudaMemsetAsync(p.wmax_bits, 0, Gs * 8, st));
    int grid = (B + 7) / 8;                                   // per trainer, as a stand-alone learner picks it
    if (grid > num_sms() * 4) grid = num_sms() * 4;
    // n_entries: the trainer's own transition count (every trainer holds the same number)
    per_sample_kernel<<<dim3(grid, p.G), 256, 0, st>>>(p, B, u_tape, seed ^ kPerSalt, per.calls++, (double)(count / G), p.beta,
                                                       slot_out ? slot_out : p.idx, p.w_raw, p.wmax_bits);
    UAVRL_LAUNCHED();
    per_norm_kernel<<<dim3((B + 255) / 256, p.G), 256, 0, st>>>(B, p.w_raw, p.wmax_bits, w_out ? w_out : p.w);
    UAVRL_LAUNCHED();
    return 0;
}

BatchSrc ReplayStore::per_source(uint64_t seed, int B, const BatchSrc &src_in, cudaStream_t st, int *rc)
{
    BatchSrc src = src_in;
    if ((*rc = per_sample(seed, B, nullptr, nullptr, nullptr, st))) return src;
    // grouped learner: [G][B] trainer-local slots, weights and errors; trainer_src hands trainer g its row of each
    const PerDev &p = per.dev;
    src.idx_tape = p.idx; src.idx_is_slot = 1; src.is_w = p.w; src.abs_err = p.abs_err;
    return src;
}

int per_entry_set(ReplayStore *rs, int device, int32_t n, const int32_t *slots, const double *prio, const float *abs_err, int32_t clip,
                  cudaStream_t st)
{
    if (!rs || !rs->per_enabled() || n <= 0 || !slots || (!prio && !abs_err))
        return fail(UAVRL_ERR_INVALID, "bad argument / prioritised replay not enabled");
    UAVRL_CUDA(cudaSetDevice(device));
    return rs->per_set(n, slots, prio, abs_err, clip, st);
}

int per_entry_sample(ReplayStore *rs, int device, uint64_t seed, int32_t B, const double *u_tape, int32_t *slots, float *w, cudaStream_t st)
{
    if (!rs || !rs->per_enabled() || B <= 0 || !slots || !w) return fail(UAVRL_ERR_INVALID, "bad argument / prioritised replay not enabled");
    if (rs->count <= 0) return fail(UAVRL_ERR_STATE, "the replay is empty");
    UAVRL_CUDA(cudaSetDevice(device));
    return rs->per_sample(seed, B, u_tape, slots, w, st);
}

int per_entry_get(ReplayStore *rs, int device, double *leaves, double *total, double *beta)
{
    if (!rs || !rs->per_enabled()) return fail(UAVRL_ERR_INVALID, "prioritised replay not enabled");
    UAVRL_CUDA(cudaSetDevice(device));
    return rs->per_get(leaves, total, beta);
}

int ReplayStore::per_get(double *leaves_host, double *total_out, double *beta_out) const
{
    UAVRL_CUDA(cudaDeviceSynchronize());
    const PerDev &p = per.dev;
    const size_t Gs = (size_t)p.G;
    if (leaves_host) UAVRL_CUDA(cudaMemcpy(leaves_host, p.leaf, Gs * p.cap * 8, cudaMemcpyDeviceToHost));
    if (total_out) {                                              // [G]: each tree's l2 entries summed in order
        std::vector<double> h(Gs * p.n2);
        UAVRL_CUDA(cudaMemcpy(h.data(), p.l2, Gs * p.n2 * 8, cudaMemcpyDeviceToHost));
        for (size_t g = 0; g < Gs; ++g) {
            double s = 0.0;
            for (int64_t k = 0; k < p.n2; ++k) s += h[g * p.n2 + k];
            total_out[g] = s;
        }
    }
    if (beta_out) *beta_out = p.beta;
    return 0;
}

int ReplayStore::per_clear()
{
    if (!per.dev.enabled) return 0;
    UAVRL_CUDA(cudaDeviceSynchronize());
    const PerDev &p = per.dev;
    const size_t Gs = (size_t)p.G;                                // every trainer's tree
    UAVRL_CUDA(cudaMemset(p.leaf, 0, Gs * p.cap * 8));
    UAVRL_CUDA(cudaMemset(p.l1, 0, Gs * p.n1 * 8));
    UAVRL_CUDA(cudaMemset(p.l2, 0, Gs * p.n2 * 8));
    return 0;
}

}  // namespace uavrl
