// per.cu -- prioritised replay kernels + C ABI (design in per.cuh).
#include "per.cuh"

#include <math.h>

#include <vector>

#include "learner.cuh"

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
__global__ void per_leaf_kernel(PerDev p, int n, const int32_t *__restrict__ slots, int64_t first, const double *__restrict__ prio,
                                const float *__restrict__ err, int mode, double fill, int n_first, double fill_rest)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t s = slots ? (int64_t)slots[i] : (first + i) % p.cap;
    double v;
    if (mode == 0) v = prio ? prio[i] : (i < n_first ? fill : fill_rest);
    else {
        float e = fabsf(err[i]) + (float)p.eps;
        if (mode == 2) e = fminf(e, (float)p.err_upper);
        v = (double)powf(e, (float)p.alpha);
    }
    p.leaf[s] = v;
}

// one warp per touched slot: recompute the l1 entry (level 1) or the l2 entry (level 2) that covers it
__global__ void per_level_kernel(PerDev p, int n, const int32_t *__restrict__ slots, int64_t first, int level)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    const int64_t s = slots ? (int64_t)slots[w] : (first + w) % p.cap;
    const int64_t pos = per_pos(p, s);
    if (level == 1) {
        const int64_t g = pos >> 5, j = (g << 5) + lane;
        const double x = j < p.cap ? p.leaf[per_slot(p, j)] : 0.0;
        const double sum = warp_sum(x);
        if (lane == 0) p.l1[g] = sum;
    } else {
        const int64_t b = pos >> 10, j = (b << 5) + lane;
        const double x = j < p.n1 ? p.l1[j] : 0.0;
        const double sum = warp_sum(x);
        if (lane == 0) p.l2[b] = sum;
    }
}

// ---- ReplayTree.sample2 (:186-213)
__global__ void __launch_bounds__(256) per_sample_kernel(PerDev p, int B, const double *__restrict__ u_tape, uint64_t key, uint64_t call,
                                                         double n_entries, double beta, int32_t *__restrict__ slot_out,
                                                         double *__restrict__ w_raw, unsigned long long *wmax_bits)
{
    __shared__ double pre[kPerMaxL2];       // inclusive prefix of l2
    __shared__ double wsum[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
    if (i < B) w[i] = (float)(w_raw[i] / __longlong_as_double((long long)*wmax_bits));      // :210
}

static int per_refresh(uavrl_learner *l, int n, const int32_t *slots, int64_t first, cudaStream_t st)
{
    const PerDev &p = l->per;
    const int blocks = (int)(((int64_t)n * 32 + 255) / 256);
    per_level_kernel<<<blocks, 256, 0, st>>>(p, n, slots, first, 1);
    UAVRL_LAUNCHED();
    per_level_kernel<<<blocks, 256, 0, st>>>(p, n, slots, first, 2);
    UAVRL_LAUNCHED();
    l->pdl_prev = kPdlNone;
    return 0;
}

int per_fill_range(uavrl_learner *l, int64_t first_slot, int64_t n, double value, cudaStream_t st, int64_t n_first, double value_rest)
{
    if (n <= 0) return 0;
    per_leaf_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(l->per, (int)n, nullptr, first_slot % l->per.cap, nullptr, nullptr, 0, value,
                                                          (int)(n_first < 0 ? n : n_first), value_rest);
    UAVRL_LAUNCHED();
    return per_refresh(l, (int)n, nullptr, first_slot % l->per.cap, st);
}

int per_set(uavrl_learner *l, int n, const int32_t *slots, const double *prio, const float *abs_err, int clip, cudaStream_t st)
{
    per_leaf_kernel<<<(n + 255) / 256, 256, 0, st>>>(l->per, n, slots, 0, prio, abs_err, prio ? 0 : (clip ? 2 : 1), 0.0, n, 0.0);
    UAVRL_LAUNCHED();
    return per_refresh(l, n, slots, 0, st);
}

int per_sample(uavrl_learner *l, int B, const double *u_tape, int32_t *slot_out, float *w_out, cudaStream_t st)
{
    PerDev &p = l->per;
    if (B > p.scratch_cap) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        cudaFree(p.idx); cudaFree(p.w); cudaFree(p.abs_err); cudaFree(p.w_raw);
        UAVRL_CUDA(cudaMalloc((void **)&p.idx, (size_t)B * 4));
        UAVRL_CUDA(cudaMalloc((void **)&p.w, (size_t)B * 4));
        UAVRL_CUDA(cudaMalloc((void **)&p.abs_err, (size_t)B * 4));
        UAVRL_CUDA(cudaMalloc((void **)&p.w_raw, (size_t)B * 8));
        p.scratch_cap = B;
    }
    p.beta = fmin(1.0, p.beta + p.beta_inc);                  // :195
    UAVRL_CUDA(cudaMemsetAsync(p.wmax_bits, 0, 8, st));
    int grid = (B + 7) / 8;
    if (grid > num_sms() * 4) grid = num_sms() * 4;
    per_sample_kernel<<<grid, 256, 0, st>>>(p, B, u_tape, l->cfg.seed ^ 0x9E12ull, l->per_calls++, (double)l->count, p.beta,
                                          slot_out ? slot_out : p.idx, p.w_raw, p.wmax_bits);
    UAVRL_LAUNCHED();
    per_norm_kernel<<<(B + 255) / 256, 256, 0, st>>>(B, p.w_raw, p.wmax_bits, w_out ? w_out : p.w);
    UAVRL_LAUNCHED();
    l->pdl_prev = kPdlNone;
    return 0;
}

void per_free(uavrl_learner *l)
{
    PerDev &p = l->per;
    if (!p.enabled) return;
    cudaFree(p.leaf); cudaFree(p.l1); cudaFree(p.l2); cudaFree(p.idx); cudaFree(p.w); cudaFree(p.abs_err); cudaFree(p.w_raw);
    cudaFree(p.wmax_bits);
    memset(&p, 0, sizeof(p));
}

}  // namespace uavrl

using namespace uavrl;

extern "C" {

int uavrl_per_enable(uavrl_learner *l, double alpha, double beta0, double beta_inc, double eps, double err_upper)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (l->G > 1) return fail(UAVRL_ERR_INVALID, "prioritised replay is not available on a learner with several trainers");
    if (l->per.enabled) return fail(UAVRL_ERR_STATE, "prioritised replay is already enabled");
    if (l->count != 0) return fail(UAVRL_ERR_STATE, "enable prioritised replay before the first transition is stored");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    PerDev &p = l->per;
    memset(&p, 0, sizeof(p));
    p.cap = l->slots;
    int64_t pow2 = 1;
    while (pow2 < p.cap) pow2 <<= 1;
    p.rot = pow2 - p.cap;
    p.n1 = (p.cap + 31) / 32; p.n2 = (p.n1 + 31) / 32;
    if (p.n2 > kPerMaxL2) return fail(UAVRL_ERR_INVALID, "prioritised replay supports at most 4194304 slots");
    p.alpha = alpha >= 0 ? alpha : 0.6; p.beta = beta0 >= 0 ? beta0 : 0.4; p.beta_inc = beta_inc >= 0 ? beta_inc : 0.001;   // :141-148
    p.eps = eps >= 0 ? eps : 0.01; p.err_upper = err_upper >= 0 ? err_upper : 1.0;
    int rc;
    if ((rc = dev_alloc(&p.leaf, (size_t)p.cap)) || (rc = dev_alloc(&p.l1, (size_t)p.n1)) || (rc = dev_alloc(&p.l2, (size_t)p.n2)) ||
        (rc = dev_alloc(&p.wmax_bits, 1)))
        return rc;
    p.enabled = 1;
    return 0;
}

int uavrl_per_set_priorities(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const double *prio_dev, void *stream)
{
    if (!l || !l->per.enabled || n <= 0 || !slots_dev || !prio_dev) return fail(UAVRL_ERR_INVALID, "bad argument / prioritised replay not enabled");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return per_set(l, n, slots_dev, prio_dev, nullptr, 0, (cudaStream_t)stream);
}

int uavrl_per_set_errors(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const float *abs_err_dev, int32_t clip, void *stream)
{
    if (!l || !l->per.enabled || n <= 0 || !slots_dev || !abs_err_dev) return fail(UAVRL_ERR_INVALID, "bad argument / prioritised replay not enabled");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return per_set(l, n, slots_dev, nullptr, abs_err_dev, clip, (cudaStream_t)stream);
}

int uavrl_per_sample(uavrl_learner *l, int32_t B, const double *u_tape_dev, int32_t *slots_out_dev, float *weights_out_dev, void *stream)
{
    if (!l || !l->per.enabled || B <= 0 || !slots_out_dev || !weights_out_dev) return fail(UAVRL_ERR_INVALID, "bad argument / prioritised replay not enabled");
    if (l->count <= 0) return fail(UAVRL_ERR_STATE, "the replay is empty");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return per_sample(l, B, u_tape_dev, slots_out_dev, weights_out_dev, (cudaStream_t)stream);
}

int uavrl_per_get(uavrl_learner *l, double *leaves_host, double *total_out, double *beta_out)
{
    if (!l || !l->per.enabled) return fail(UAVRL_ERR_INVALID, "prioritised replay not enabled");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const PerDev &p = l->per;
    if (leaves_host) UAVRL_CUDA(cudaMemcpy(leaves_host, p.leaf, (size_t)p.cap * 8, cudaMemcpyDeviceToHost));
    if (total_out) {
        std::vector<double> h((size_t)p.n2);
        UAVRL_CUDA(cudaMemcpy(h.data(), p.l2, (size_t)p.n2 * 8, cudaMemcpyDeviceToHost));
        double s = 0.0;
        for (double x : h) s += x;
        *total_out = s;
    }
    if (beta_out) *beta_out = p.beta;
    return 0;
}

}  // extern "C"
