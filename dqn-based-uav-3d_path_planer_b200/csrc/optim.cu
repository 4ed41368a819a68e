// optim.cu -- the optimiser step of both learners (reduce_adam_kernel: reduce the gradient partials in a fixed order, Adam,
// hard target copy, weight-image refresh) and its data-parallel form (dp_allreduce_adam_kernel: the same step fused with a
// one-shot NVLink all-reduce over the ranks' symmetric receive buffers), with the CUDA IPC setup of those buffers.  sm_90a.
//
// Replaces (SURVEY.md K7): torch.optim.Adam step + hard_update (DuelingDQN_Trainer.py:176-184,199-202), and SAC_Trainer's
// Adam steps (SAC_Trainer.py:42-44,55).
#include "optim.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>

namespace uavrl {

// ------------------------------------------------------------------ reduce partials + Adam + target copy

// 64 parameters per CTA x 4 partial-groups: the cross-CTA gradient reduction runs 4-wide with
// independent loads in flight, then Adam; fixed summation order -> run-to-run deterministic.
// One __restrict__ parameter per pointer (launch_reduce_adam unpacks an AdamPtrs into them): only __restrict__ kernel parameters
// let the compiler read the partials, moments and maps through the read-only path -- __restrict__ copies inside the kernel do
// not survive the memory clobber of the PDL wait.  Taking an AdamPtrs instead made the three SAC optimiser steps 52 us per
// iteration instead of 38 us (H100 80GB HBM3, 700 W).
__global__ void __launch_bounds__(256)
reduce_adam_kernel(AdamArgs a, const float *__restrict__ partials, const float *__restrict__ loss_partials,
                   float *__restrict__ grad, float *__restrict__ local, float *__restrict__ m, float *__restrict__ v,
                   float *__restrict__ target, float *__restrict__ img_local, float *__restrict__ img_target,
                   const int32_t *__restrict__ img_map, float *__restrict__ tc_local, float *__restrict__ tc_target,
                   const int32_t *__restrict__ tc_hi, const int32_t *__restrict__ tc_lo, const int32_t *__restrict__ tc_hi2,
                   const int32_t *__restrict__ tc_lo2, float *__restrict__ loss_out)
{
    __shared__ float red[4][64];
    const int ix = threadIdx.x & 63, cg = threadIdx.x >> 6;
    const int i = blockIdx.x * 64 + ix;
    {   // trainer blockIdx.y of a grouped learner: its partials [nparts][P], vectors [P], images and loss
        const size_t g = blockIdx.y, gp = g * (size_t)a.P;
        partials += gp * (size_t)a.nparts; loss_partials += g * (size_t)a.n_loss_parts;
        grad += gp; local += gp; m += gp; v += gp; target += gp;
        img_local += g * (size_t)a.img_floats; img_target += g * (size_t)a.img_floats;
        if (tc_local) { tc_local += g * (size_t)a.tc_floats; tc_target += g * (size_t)a.tc_floats; }
        if (loss_out) loss_out += g;
    }
    AdamPtrs q;
    q.partials = partials; q.loss_partials = loss_partials; q.grad = grad; q.local = local; q.m = m; q.v = v; q.target = target;
    q.img_local = img_local; q.img_target = img_target; q.img_map = img_map; q.tc_local = tc_local; q.tc_target = tc_target;
    q.tc_hi = tc_hi; q.tc_lo = tc_lo; q.tc_hi2 = tc_hi2; q.tc_lo2 = tc_lo2; q.loss_out = loss_out;
    const bool mine = cg == 0 && i < a.P && a.apply;
    AdamPre pre;
    if (mine) pre = adam_prefetch(q, i);                 // moments, parameter, image indices: not the predecessor's output
    pdl_wait();                 // PDL (common.cuh): the gradient partials come from the predecessor
    pdl_trigger();
    float g = 0.f;
    if (i < a.P && a.nparts > 0) g = reduce_group(partials, a.P, a.nparts, i, cg);   // partials are L2 resident, latency bound
    red[cg][ix] = g;
    __syncthreads();
    if (cg == 0 && i < a.P) {
        if (a.nparts > 0) {
            g = (red[0][ix] + red[1][ix]) + (red[2][ix] + red[3][ix]);
            grad[i] = g;
        } else {
            g = grad[i];                                  // already reduced (and all-reduced) by the caller
        }
        if (mine) adam_update_pre(a, q, i, g, pre);
    }
    if (blockIdx.x == 0 && threadIdx.x >= 224 && loss_out && a.nparts > 0) {     // last warp: loss = sum / B
        const int lane = threadIdx.x & 31;
        float s = 0.f;
        for (int c = lane; c < a.n_loss_parts; c += 32) s += loss_partials[c];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) *loss_out = s * a.inv_b;
    }
}

// blocks of either optimiser kernel for a network of P parameters: each block owns 64 of them
static unsigned adam_blocks(int P) { return (unsigned)(P + 63) / 64; }

cudaError_t launch_reduce_adam(int G, cudaStream_t st, bool pdl, const AdamArgs &a, const AdamPtrs &q)
{
    return launch_kernel(reduce_adam_kernel, dim3(adam_blocks(a.P), G), dim3(256), 0, st, pdl, a, q.partials, q.loss_partials, q.grad,
                         q.local, q.m, q.v, q.target, q.img_local, q.img_target, q.img_map, q.tc_local, q.tc_target, q.tc_hi, q.tc_lo,
                         q.tc_hi2, q.tc_lo2, q.loss_out);
}

void adam_hyper(AdamArgs &a, float lr, int64_t t)
{
    const double b1 = 0.9, b2 = 0.999;
    const double bc1 = 1.0 - pow(b1, (double)t), bc2 = 1.0 - pow(b2, (double)t);
    a.step_size = (float)((double)lr / bc1);
    a.beta1_c = (float)(1.0 - b1); a.beta2 = (float)b2; a.beta2_c = (float)(1.0 - b2);
    a.eps = 1e-8f; a.bc2_sqrt = (float)sqrt(bc2);
}

// ---- data-parallel optimiser step: one-shot NVLink all-reduce fused with Adam, in ONE kernel, block by block, with no fence
// and no flag words.  Every rank owns a symmetric receive buffer (slot q belongs to rank q); block b owns 64 parameters of
// one network of the exchange (DpExchange: up to two networks, by block range).  It reduces its slice of this rank's
// partials and pushes each value into slot `rank` of every rank's receive buffer as ONE 8-byte word {tag : value} (a
// single-copy-atomic store: the value can never be seen without its tag -- the "LL" idea of NCCL's low-latency protocol).
// Then the 64 threads of the block poll -- in local memory -- the `world` words of their own parameter until every tag
// matches, sum the values in rank order and apply Adam.  The exchange's scalar words (a loss share, an update's stat sums)
// travel the same way from block 0.  A __threadfence_system() between data and a flag would cost a system-scope fence per
// launch even on one GPU; here nothing orders two stores, so nothing needs a fence.
// The buffer alternates halves by the parity of the tag, which advances once per exchange (an update may make several: a SAC
// update exchanges its critics, then its actor).  A rank writes exchange e + 2 into exchange e's half only after its own
// exchange e + 1 kernel has completed; completing e + 1 needs every rank's e + 1 words, and each rank pushes those only after
// its own exchange-e kernel -- the last reader of e's half on that rank -- has finished.  So no word is overwritten before
// its reader has summed it, whatever the exchanges carry.
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// sum over ranks (fixed order: every rank computes the same bits) of the words {tag : value} at recv[w * stride]
__device__ __forceinline__ float ll_gather_sum(const unsigned long long *recv, size_t stride, int world, unsigned epoch)
{
    float gsum = 0.f;
    for (int w0 = 0; w0 < world; w0 += 8) {
        unsigned long long t[8];
        bool ok;
        do {
            ok = true;
#pragma unroll
            for (int u = 0; u < 8; ++u) t[u] = (w0 + u < world) ? ld_relaxed_sys_u64(recv + (size_t)(w0 + u) * stride) : 0ull;
#pragma unroll
            for (int u = 0; u < 8; ++u) ok = ok && (w0 + u >= world || (unsigned)(t[u] >> 32) == epoch);
        } while (!ok);
#pragma unroll
        for (int u = 0; u < 8; ++u) if (w0 + u < world) gsum += __uint_as_float((unsigned)t[u]);
    }
    return gsum;
}

// partials0 / partials1 / extra_parts: the segments' and the scalar words' partials of x, as __restrict__ kernel parameters
// (reduce_adam_kernel says why)
__global__ void __launch_bounds__(256)
dp_allreduce_adam_kernel(AdamArgs a, DpExchange x, const float *__restrict__ partials0, const float *__restrict__ partials1,
                         const float *__restrict__ extra_parts, unsigned long long *const *peer_recv,
                         const unsigned long long *recv_local, size_t stride, size_t parity_off, int rank, unsigned epoch,
                         unsigned long long *trace)
{
    // trace (UAVRL_DP_TRACE=1): block 0 accumulates nanoseconds spent in {reduce, push, wait for the peers' words, Adam} and a launch count
    unsigned long long t0 = 0, t1 = 0, t2 = 0, t3 = 0;
    auto now = [] { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };
    __shared__ float red[4][64];
    const int sg = (x.n_seg > 1 && (int)blockIdx.x >= x.seg[0].blocks) ? 1 : 0;
    const int P = sg ? x.seg[1].P : x.seg[0].P, nparts = sg ? x.seg[1].nparts : x.seg[0].nparts;
    const float *partials = sg ? partials1 : partials0;
    const size_t woff = sg ? (size_t)x.seg[0].P : 0;                 // the segment's first word in a rank's slot
    const int ix = threadIdx.x & 63, cg = threadIdx.x >> 6;
    const int i = ((int)blockIdx.x - (sg ? x.seg[0].blocks : 0)) * 64 + ix;
    AdamPre pre;
    if (cg == 0 && i < P) pre = adam_prefetch(sg ? x.seg[1].q : x.seg[0].q, i);     // before the wait: nothing here is the predecessor's output
    pdl_wait();                 // PDL (common.cuh): the gradient partials come from the predecessor
    pdl_trigger();
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t0 = now();
    float g = 0.f;
    if (i < P) g = reduce_group(partials, P, nparts, i, cg);
    red[cg][ix] = g;
    __syncthreads();
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t1 = now();
    const size_t slot = parity_off + (size_t)rank * stride;
    const unsigned long long tag = (unsigned long long)epoch << 32;
    if (i < P) {
        const float gs = (red[0][ix] + red[1][ix]) + (red[2][ix] + red[3][ix]);
        for (int w = cg; w < a.world; w += 4) st_relaxed_sys_u64(peer_recv[w] + slot + woff + i, tag | __float_as_uint(gs));   // 512 contiguous bytes per peer
    }
    const size_t xoff = (size_t)x.seg[0].P + (x.n_seg > 1 ? (size_t)x.seg[1].P : 0);   // the scalar words follow the segments
    if (blockIdx.x == 0 && threadIdx.x >= 224) {                 // last warp of block 0: this rank's scalar words
#pragma unroll
        for (int j = 0; j < kDpMaxExtra; ++j) {
            if (j >= x.n_extra) break;
            const float s = warp_column_sum(extra_parts, x.n_extra_parts, x.extra_stride, j);
            if ((threadIdx.x & 31) == 0)
                for (int w = 0; w < a.world; ++w) st_relaxed_sys_u64(peer_recv[w] + slot + xoff + j, tag | __float_as_uint(s * x.extra_scale));
        }
    }
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t2 = now();
    const unsigned long long *recv = recv_local + parity_off;
    if (cg == 0 && i < P) {
        const float gsum = ll_gather_sum(recv + woff + i, stride, a.world, epoch);
        if (trace && blockIdx.x == 0 && threadIdx.x == 0) t3 = now();
        const AdamPtrs &q = sg ? x.seg[1].q : x.seg[0].q;
        q.grad[i] = gsum;
        adam_update_pre(a, q, i, gsum, pre);
    }
    if (blockIdx.x == 0 && threadIdx.x >= 256 - x.n_extra && x.extra_out) {
        const int j = 255 - threadIdx.x;
        x.extra_out[j] = ll_gather_sum(recv + xoff + j, stride, a.world, epoch);
    }
    if (trace && blockIdx.x == 0) {
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long t4 = now();
            trace[0] += t1 - t0; trace[1] += t2 - t1; trace[2] += t3 - t2; trace[3] += t4 - t3; trace[4] += 1;
        }
    }
}

cudaError_t launch_dp_exchange(PeerComm &c, const AdamArgs &a, const DpExchange &x_in, cudaStream_t st, bool pdl)
{
    DpExchange x = x_in;
    for (int k = 0; k < x.n_seg; ++k) x.seg[k].blocks = (int)adam_blocks(x.seg[k].P);
    c.tag += 1;
    const size_t stride = (size_t)x.seg[0].P + (x.n_seg > 1 ? (size_t)x.seg[1].P : 0) + (size_t)x.n_extra;   // this exchange's slot
    const size_t parity_off = (size_t)(c.tag & 1u) * (size_t)c.world * c.words;
    const int blocks = x.seg[0].blocks + (x.n_seg > 1 ? x.seg[1].blocks : 0);
    return launch_kernel(dp_allreduce_adam_kernel, dim3(blocks), dim3(256), 0, st, pdl, a, x, x.seg[0].partials,
                         x.n_seg > 1 ? x.seg[1].partials : nullptr, x.extra_parts, (unsigned long long *const *)c.peer_dev,
                         (const unsigned long long *)c.recv, stride, parity_off, (int)c.rank, c.tag, c.trace);
}

// ------------------------------------------------------------------ the data-parallel exchange's buffers (PeerComm)
PeerComm::~PeerComm()
{
    if (trace) {
        unsigned long long h[5] = { 0, 0, 0, 0, 0 };
        cudaMemcpy(h, trace, sizeof(h), cudaMemcpyDeviceToHost);
        if (h[4]) fprintf(stderr, "[dp_trace] rank %d/%d: %llu launches, block 0 mean ns: reduce %.0f  push %.0f  wait for peers' words %.0f  adam %.0f\n",
                          rank, world, h[4], (double)h[0] / h[4], (double)h[1] / h[4], (double)h[2] / h[4], (double)h[3] / h[4]);
    }
    for (int q = 0; q < world && ready; ++q)
        if (q != rank && peer_host[q]) cudaIpcCloseMemHandle(peer_host[q]);
}

constexpr size_t kBusIdBytes = 64;

int comm_init(PeerComm &c, int device, int32_t rank, int32_t world, size_t words, void *handle_out, bool bus_id)
{
    if (world < 1 || world > PeerComm::kMaxWorld || rank < 0 || rank >= world || !handle_out)
        return fail(UAVRL_ERR_INVALID, "bad rank/world/handle pointer");
    UAVRL_CUDA(cudaSetDevice(device));
    if (!c.recv || c.recv_world != world || c.words != words) {   // first call, or re-initialised with another size
        // recv[2][world][words] words of 8 bytes {tag : value} (tag 0 = never written)
        DevMem m;
        unsigned long long *recv = nullptr;
        if (int rc = m.alloc(recv, 2 * (size_t)world * words)) return rc;
        UAVRL_CUDA(cudaDeviceSynchronize());                     // nothing may still use the buffer being replaced
        c.recv_mem = std::move(m);
        c.recv = recv; c.recv_world = world; c.words = words;
    }
    c.rank = rank; c.world = world;
    cudaIpcMemHandle_t hg;
    UAVRL_CUDA(cudaIpcGetMemHandle(&hg, c.recv));
    memcpy(handle_out, &hg, sizeof(hg));
    if (bus_id) {
        char id[kBusIdBytes] = { 0 };
        UAVRL_CUDA(cudaDeviceGetPCIBusId(id, (int)kBusIdBytes - 1, device));
        memcpy((char *)handle_out + sizeof(hg), id, kBusIdBytes);
    }
    return 0;
}

int comm_connect(PeerComm &c, int device, const void *handles, bool bus_id)
{
    UAVRL_CUDA(cudaSetDevice(device));
    const size_t rec = sizeof(cudaIpcMemHandle_t) + (bus_id ? kBusIdBytes : 0);
    if (bus_id) {                               // every rank's device must differ from every other's: checked before any handle opens
        for (int q = 0; q < c.world; ++q)
            for (int p = 0; p < q; ++p)
                if (!memcmp((const char *)handles + p * rec + sizeof(cudaIpcMemHandle_t),
                            (const char *)handles + q * rec + sizeof(cudaIpcMemHandle_t), kBusIdBytes))
                    return fail(UAVRL_ERR_INVALID, "ranks " + std::to_string(p) + " and " + std::to_string(q) +
                                                       " share one device: each rank of the exchange needs its own GPU");
    }
    for (int q = 0; q < c.world; ++q) {
        if (q == c.rank) { c.peer_host[q] = c.recv; continue; }
        cudaIpcMemHandle_t hg;
        memcpy(&hg, (const char *)handles + (size_t)q * rec, sizeof(hg));
        UAVRL_CUDA(cudaIpcOpenMemHandle(&c.peer_host[q], hg, cudaIpcMemLazyEnablePeerAccess));
    }
    DevMem m;
    unsigned long long **table = nullptr;
    if (int rc = m.alloc(table, (size_t)c.world, false)) return rc;
    UAVRL_CUDA(cudaMemcpy(table, c.peer_host, sizeof(void *) * c.world, cudaMemcpyHostToDevice));
    c.peer_mem = std::move(m);                                   // cudaFree of the old table waits for the device
    c.peer_dev = table;
    static const bool trace = getenv("UAVRL_DP_TRACE") != nullptr;
    if (trace && !c.trace)
        if (int rc = c.trace_mem.alloc(c.trace, 5)) return rc;
    c.ready = true;
    return 0;
}

}  // namespace uavrl
