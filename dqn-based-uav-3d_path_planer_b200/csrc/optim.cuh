// optim.cuh -- the optimiser step both learners launch (reduce_adam_kernel) and the data-parallel exchange they share
// (dp_allreduce_adam_kernel and its symmetric receive buffers, PeerComm); optim.cu holds the kernels and the host side.
#pragma once
#include "common.cuh"

namespace uavrl {

// optimiser kernel arguments (reduce_adam_kernel, dp_allreduce_adam_kernel)
struct AdamArgs {
    int P, nparts, apply, hard, world, n_loss_parts;
    int img_floats, tc_floats;        // grouped learner (gridDim.y = G): per-trainer strides of the fp32 / tensor-core weight images
    float step_size, beta1_c, beta2, beta2_c, eps, bc2_sqrt, inv_b;
};

// everything the optimiser step reads / writes (flat state_dict-ordered vectors + the kernel-layout weight images)
struct AdamPtrs {
    const float *partials, *loss_partials;
    float *grad, *local, *m, *v, *target, *img_local, *img_target;
    const int32_t *img_map;
    float *tc_local, *tc_target;
    const int32_t *tc_hi, *tc_lo, *tc_hi2, *tc_lo2;
    float *loss_out;
};

#if defined(__CUDACC__)
// Partial-gradient reduction in a FIXED order (run-to-run deterministic, and the same whichever kernel performs it):
// partial c belongs to group c % 4; a group keeps 8 accumulators (8 independent loads in flight per pass over 32 partials);
// the total is (g0 + g1) + (g2 + g3).
__device__ __forceinline__ float reduce_group(const float *__restrict__ partials, int P, int nparts, int i, int cg)
{
    float acc[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = 0.f;
    int c = cg;
    for (; c + 28 < nparts; c += 32) {
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] += partials[(size_t)(c + 4 * u) * P + i];
    }
    for (; c < nparts; c += 4) acc[0] += partials[(size_t)c * P + i];
    return ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
}

__device__ __forceinline__ void tf32_split_f(float x, float &hi, float &lo)
{
    hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);     // = cvt.rna.tf32.f32 for finite x (wgmma.cuh: tf32_split)
    lo = x - hi;
}

// torch.optim.Adam single-tensor step for parameter i with gradient g (lerp, mul/addcmul, sqrt/div/add, addcdiv), the hard
// target update (DuelingDQN_Trainer.py:199-202) and the refresh of the fp32 and tensor-core weight images
// what the step reads besides the gradient: nothing a gradient-producing predecessor writes, so an optimiser kernel launched
// programmatically behind one fetches it BEFORE griddepcontrol.wait (one memory round trip off the post-wait chain)
struct AdamPre { float m, v, p; int im, ih, il, ih2, il2; };
__device__ __forceinline__ AdamPre adam_prefetch(const AdamPtrs &q, int i)
{
    AdamPre r;
    r.m = q.m[i]; r.v = q.v[i]; r.p = q.local[i]; r.im = q.img_map[i];
    r.ih = r.il = r.ih2 = r.il2 = -1;
    if (q.tc_local) { r.ih = q.tc_hi[i]; r.il = q.tc_lo[i]; r.ih2 = q.tc_hi2[i]; r.il2 = q.tc_lo2[i]; }
    return r;
}
__device__ __forceinline__ void adam_update_pre(const AdamArgs &a, const AdamPtrs &q, int i, float g, const AdamPre &pre)
{
    // every operation individually rounded (no FMA contraction): the optimiser kernels that share this function
    // (reduce_adam_kernel, dp_allreduce_adam_kernel) then produce bit-identical parameters by construction
    float mi = pre.m, vi = pre.v, p = pre.p;
    mi = __fadd_rn(mi, __fmul_rn(__fsub_rn(g, mi), a.beta1_c));                                  // exp_avg.lerp_(grad, 1 - beta1)
    vi = __fadd_rn(__fmul_rn(vi, a.beta2), __fmul_rn(__fmul_rn(a.beta2_c, g), g));               // exp_avg_sq.mul_(beta2).addcmul_(g, g, 1 - beta2)
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), a.bc2_sqrt), a.eps);                 // (sqrt(v) / sqrt(bc2)).add_(eps)
    p = __fsub_rn(p, __fmul_rn(a.step_size, __fdiv_rn(mi, denom)));                              // param.addcdiv_(m, denom, -step_size)
    q.m[i] = mi; q.v[i] = vi; q.local[i] = p;
    const int im = pre.im;
    q.img_local[im] = p;
    if (a.hard) { q.target[i] = p; q.img_target[im] = p; }
    if (q.tc_local) {                                        // tensor-core images: TF32 hi/lo split of the new value
        const int ih = pre.ih, il = pre.il;
        float hi = p, lo = 0.f;
        if (il >= 0) tf32_split_f(p, hi, lo);
        q.tc_local[ih] = hi;
        if (il >= 0) q.tc_local[il] = lo;
        const int ih2 = pre.ih2, il2 = pre.il2;
        if (ih2 >= 0) { q.tc_local[ih2] = hi; q.tc_local[il2] = lo; }
        if (a.hard) {
            q.tc_target[ih] = hi;
            if (il >= 0) q.tc_target[il] = lo;
            if (ih2 >= 0) { q.tc_target[ih2] = hi; q.tc_target[il2] = lo; }
        }
    }
}

// Sum of column j of n rows of `stride` floats, the order every scalar partial sum of an update takes: lane l adds rows l,
// l + 32, ... in turn, then a butterfly over the warp.  Every lane of the (full) warp calls it and receives the sum.
__device__ __forceinline__ float warp_column_sum(const float *p, int n, int stride, int j)
{
    float s = 0.f;
    for (int c = threadIdx.x & 31; c < n; c += 32) s += p[(size_t)c * stride + j];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    return s;
}
#endif

// reduce_adam_kernel on the G trainers' vectors (gridDim.y = G) with the pointers of q; pdl: programmatic dependent launch
cudaError_t launch_reduce_adam(int G, cudaStream_t st, bool pdl, const AdamArgs &a, const AdamPtrs &q);

// torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8) at step t with learning rate lr: the fields of AdamArgs the step computes in
// double precision on the host (bias corrections, step size)
void adam_hyper(AdamArgs &a, float lr, int64_t t);

// One rank's side of the data-parallel exchange (dp_allreduce_adam_kernel): its symmetric receive buffer recv[2][world][words]
// of 8-byte words {exchange tag : value}, where slot q is written by rank q with remote stores, and every rank's buffer as
// mapped on this device.  Both learners own one (uavrl_learner_comm_*, uavrl_sac_comm_*).
struct PeerComm {
    static constexpr int kMaxWorld = 64;
    int32_t rank = 0, world = 1;
    unsigned long long *recv = nullptr;
    int32_t recv_world = 0;           // world the buffer was sized for
    size_t words = 0;                 // words of one rank's slot: the largest exchange the owner makes
    unsigned long long **peer_dev = nullptr;    // device array [world]
    void *peer_host[kMaxWorld] = { nullptr };
    bool ready = false;               // comm_connect has run
    unsigned tag = 0;                 // tag of the latest exchange; 0 = never written
    // UAVRL_DP_TRACE=1 (set when the comm connects): block 0's summed nanoseconds in {reduce, push, wait for the peers' words,
    // Adam} and the exchange count, printed when the comm is destroyed
    unsigned long long *trace = nullptr;
    DevMem recv_mem, peer_mem, trace_mem;   // owners of recv, peer_dev and trace
    ~PeerComm();                      // prints the trace, closes the peers' mapped buffers
};
// comm_init: (re)size the receive buffer for `world` ranks of `words` words each and write its CUDA IPC handle into
// handle_out; with bus_id, the handle is followed by this device's PCI bus id (64 bytes), which comm_connect checks: two
// ranks on one device would spin forever in the exchange.  Refuses a rank outside [0, world), a world outside
// [1, kMaxWorld] and a null handle_out.  comm_connect: open every rank's handle (handles: [world] records).
int comm_init(PeerComm &c, int device, int32_t rank, int32_t world, size_t words, void *handle_out, bool bus_id);
int comm_connect(PeerComm &c, int device, const void *handles, bool bus_id);

// One exchange of dp_allreduce_adam_kernel: the optimiser steps of n_seg networks, segment k taking `blocks` blocks of 64
// parameters after segment k - 1's (launch_dp_exchange fills `blocks`) and words [sum of the earlier P, + P) of a rank's slot,
// then n_extra scalar words: column j of the [n_extra_parts][extra_stride] partials, reduced by warp_column_sum and scaled,
// summed over ranks into extra_out[j].  Every rank's slot holds the words in that order.
struct DpSeg { const float *partials; int nparts, P, blocks; AdamPtrs q; };
struct DpExchange {
    DpSeg seg[2];
    int n_seg;
    const float *extra_parts;
    int n_extra_parts, extra_stride, n_extra;
    float extra_scale;
    float *extra_out;
};
constexpr int kDpMaxExtra = 2;
// the exchange x on comm (its tag advances by one) with the Adam hyper-parameters of a
cudaError_t launch_dp_exchange(PeerComm &comm, const AdamArgs &a, const DpExchange &x, cudaStream_t st, bool pdl);

}  // namespace uavrl
