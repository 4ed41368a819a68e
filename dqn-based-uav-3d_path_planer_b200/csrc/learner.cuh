// learner.cuh -- Q-network / replay / optimiser state of one learner (device-resident) + host handle.
#pragma once
#include "common.cuh"
#include "per.cuh"
#include "replay.cuh"

namespace uavrl {

constexpr int kTile = 32;             // samples per CTA tile
constexpr int kNetThreads = 256;      // 8 warps: lane -> output unit, warp -> 4 samples
constexpr int kMaxDim = 128;          // every layer width (and in_dim) <= 128
constexpr int kMaxLayers = UAVRL_MAX_HIDDEN + 1;   // trunk layers + (combined) head
constexpr int kFedProbes = 10;        // probe states per trainer of a federation round (PathPlan_City.py:658)

// One dense layer as the kernels see it.  Weights live in smem transposed: Wt[k][o], ld = out+1
// (odd when out is even -> conflict-free whether lanes walk o or k).
struct LayerDev {
    int32_t in, out;                  // out of the head = n_actions (+1 value row when dueling)
    int32_t w_off, b_off;             // offsets in the flat state_dict-ordered parameter vector
    int32_t w2_off, b2_off;           // second head block (rows out_main..out-1): dueling fc_V, SAC actor fc_std; -1 if none
    int32_t out_main;                 // rows served by (w_off, b_off)
    int32_t smem_w, smem_b;           // offsets (floats) inside the smem weight area
};

struct NetDev {
    int32_t in_dim, n_layers, n_actions, dueling;
    int32_t P;                        // parameter count
    int32_t smem_w_floats;            // total smem floats for Wt + biases
    int32_t act_off[kMaxLayers + 1];  // smem offsets of the activation planes X0, H1.. (floats)
    int32_t act_ld[kMaxLayers + 1];
    int32_t smem_total_floats;        // whole dynamic smem carve-up for the update kernel
    LayerDev L[kMaxLayers];
};

// ---- tensor-core (wgmma) forward path: one dense layer as a B operand [N_pad][K_pad], K-major canonical
// layout (wgmma.cuh), hi and lo images of the 3xTF32 split
struct TcLayer {
    int32_t K_pad, N_pad, K_real, N_real;
    int32_t hi_off, lo_off;            // byte offsets inside the TC weight image
    int32_t bias_off;                  // float index of the zero-padded bias vector inside the image's bias area
    // transposed copy W^T as a B operand [K_pad rows][N_pad cols] for the dX chain (layers >= 1 only; -1 otherwise)
    int32_t t_hi_off, t_lo_off;
    // where this layer's pieces live in the flat parameter / gradient vector (state_dict order)
    int32_t w_off, b_off, w2_off, b2_off, out_main;
    int32_t act_off, dz_off;           // float offsets of this layer's input activations / output derivatives in the
                                       // per-sample scratch rows (act: layer input, valid for l >= 1; dz: dLoss/d(pre-activation))
};

struct TcNet {
    int32_t n_layers, in_dim, n_actions, dueling;
    int32_t img_bytes;                 // forward image: all layers hi|lo, then biases
    int32_t bias_base;                 // byte offset of the bias area
    int32_t train_img_bytes;           // forward image + transposed blocks (training chain)
    int32_t max_rows;                  // rows of the largest forward tile: 128, or 64 when 128 rows do not fit shared memory
    int32_t train_max_rows;            // rows of the largest training tile: 64, or 32 when 64 rows do not fit (tc_train_init)
    int32_t a_bytes;                   // bytes of ONE A-operand buffer (hi or lo): max_rows x max K_pad
    int32_t max_k;                     // max K_pad over layers
    int32_t act_stride, dz_stride;     // floats per sample in the activation / derivative scratch
    int32_t acc_ld;                    // floats per row of the shared-memory accumulator tile (wgmma.cuh mma_3xtf32)
    TcLayer L[kMaxLayers];
};

#if defined(__CUDACC__)
// ---- Q-head arithmetic shared by the fp32 kernels (learner.cu) and the tensor-core kernels (tc_chain.cuh).  Device code is
// compiled with FMA contraction on: each expression keeps its operand order, so both paths produce the same bits.

// TD target y = r + gamma * next_q * (1 - d)  (DQN_Trainer.py:99 / :114, DuelingDQN_Trainer.py:171)
__device__ __forceinline__ float td_target(float r, float gamma, float next_q, float d) { return r + (gamma * next_q * (1.f - d)); }

// Per-sample loss term of diff = Q(s, a) - y with the importance weight of sample b (prioritised replay; 1 without), and
// dLoss/dQ(s, a) into gq; writes |diff| for the priority update.  kind 0: MSELoss (BaseTrainer.py:40), 1: SmoothL1Loss(beta = 1)
__device__ __forceinline__ float td_loss(const BatchSrc &src, int b, float diff, int kind, float inv_global_b, float &gq)
{
    const float wb = src.is_w ? src.is_w[b] : 1.f;
    if (src.abs_err) src.abs_err[b] = fabsf(diff);
    if (kind == 0) {
        gq = (2.f * diff * wb) * inv_global_b;
        return wb * (diff * diff);
    }
    const float ad = fabsf(diff);
    gq = (fminf(fmaxf(diff, -1.f), 1.f) * wb) * inv_global_b;
    return wb * (ad < 1.f ? 0.5f * (diff * diff) : ad - 0.5f);
}

// eps-greedy draw of row `row` (DuelingDQN_Trainer.py:89-97): true = take the greedy action, else the random action ra.  The
// uniform and the random action come from the tapes at tape_row when given, else from Philox(key, call, row).
__device__ __forceinline__ bool eps_greedy(float eps, int is_train, const float *u_tape, const int32_t *rand_tape, size_t tape_row,
                                           uint64_t key, uint64_t call, int row, int n_actions, int &ra)
{
    float u;
    if (u_tape) { u = u_tape[tape_row]; ra = rand_tape ? rand_tape[tape_row] : 0; }
    else {
        uint32_t r[4];
        Philox::gen(key, call, (uint64_t)row, r);
        u = Philox::u01(r[0]);
        ra = (int)(((uint64_t)r[1] * (uint64_t)n_actions) >> 32);
    }
    return u > eps || !is_train;
}

// Federation: the loss entry of one probe group, M[p][w_set] = (sum of its kFedProbes rows' squared Q differences d2, in row
// order) / (S A); first_row = the group's first row in the [G][S] probe rows.
__device__ __forceinline__ void fed_group_loss(const float *d2, size_t first_row, int n, int w_set, int n_actions, float *loss_out)
{
    float s2 = 0.f;
    for (int r = 0; r < kFedProbes; ++r) s2 += d2[r];
    const size_t p = first_row / kFedProbes;
    loss_out[p * (size_t)(n / kFedProbes) + w_set] = s2 / (float)(kFedProbes * n_actions);
}
#endif

// One rank's side of the data-parallel exchange (dp_allreduce_adam_kernel, learner.cu): its symmetric receive buffer
// recv[2][world][words] of 8-byte words {exchange tag : value}, where slot q is written by rank q with remote stores, and every
// rank's buffer as mapped on this device.  Both learners own one (uavrl_learner_comm_*, uavrl_sac_comm_*).
struct PeerComm {
    int32_t rank = 0, world = 1;
    unsigned long long *recv = nullptr;
    int32_t recv_world = 0;           // world the buffer was sized for
    size_t words = 0;                 // words of one rank's slot: the largest exchange the owner makes
    unsigned long long **peer_dev = nullptr;    // device array [world]
    void *peer_host[64] = { nullptr };
    bool ready = false;               // comm_connect has run
    unsigned tag = 0;                 // tag of the latest exchange; 0 = never written
    DevMem recv_mem, peer_mem;        // owners of recv and peer_dev
    ~PeerComm();                      // closes the peers' mapped buffers
};
// comm_init: (re)size the receive buffer for `world` ranks of `words` words each and write its CUDA IPC handle into
// handle_out; with bus_id, the handle is followed by this device's PCI bus id (64 bytes), which comm_connect checks: two
// ranks on one device would spin forever in the exchange.  comm_connect: open every rank's handle (handles: [world] records).
int comm_init(PeerComm &c, int device, int32_t rank, int32_t world, size_t words, void *handle_out, bool bus_id);
int comm_connect(PeerComm &c, int device, const void *handles, bool bus_id);

}  // namespace uavrl

struct uavrl_learner {
    uavrl_learner_config cfg;
    uavrl::NetDev net;
    // parameters and optimiser state (flat, state_dict order)
    float *local = nullptr, *target = nullptr, *m = nullptr, *v = nullptr, *grad = nullptr;
    // kernel-layout copies of the two networks (exactly the smem weight image: transposed, padded),
    // kept in sync by the optimiser kernel so a CTA stages a whole network with one TMA bulk copy
    float *img_local = nullptr, *img_target = nullptr;
    int32_t *img_map = nullptr;       // flat parameter index -> image index
    int32_t dual_weights = 0;         // update kernel keeps local+target images resident at once
    // tensor-core forward path (act + TD target); tc_ok = the network fits the SMEM-resident wgmma kernel
    uavrl::TcNet tc;
    bool tc_ok = false;
    bool tc_fixed_fwd = false, tc_fixed_train = false;   // tc_fixed_chains(tc, false / true), set by tc_init
    bool use_tc = true;               // runtime switch (uavrl_learner_set_tensor_cores): false = fp32 CUDA-core path
    int32_t is_train = 1;             // Trainer.Is_Train for the lockstep loops (uavrl_learner_set_is_train): 0 = always greedy
    unsigned char *tc_img_local = nullptr, *tc_img_target = nullptr;
    int32_t *tc_hi_map = nullptr, *tc_lo_map = nullptr;   // flat param index -> float index in the TC image (-1: none)
    float *y_buf = nullptr;           // [batch_size] TD targets produced by the tensor-core pass
    int32_t *astar_buf = nullptr;     // [batch_size] double-DQN argmax actions
    int32_t y_cap = 0;
    // tensor-core training path scratch (per sampled transition): hidden activations and dLoss/d(pre-activation)
    int32_t *tc_hi2_map = nullptr, *tc_lo2_map = nullptr;  // flat param index -> transposed-block positions (-1: none)
    float *act_buf = nullptr, *dz_buf = nullptr;
    bool tc_train_ok = false;
    int32_t train_cap = 0;
    float *partials = nullptr;        // [max_ctas][P] per-CTA gradient partials
    float *loss_partials = nullptr;   // [max_ctas]
    float *loss_dev = nullptr;        // [G]
    int32_t max_ctas = 0;
    int32_t parts_cap = 0;            // gradient / loss partial slots per trainer (partials: [G][parts_cap][P])
    // grouped learner (uavrl_learner_create_trainers): G independent trainers of the same network.  Every per-network vector
    // and weight image is [G][...], trainer g acts for envs [g Ng, (g + 1) Ng) and samples only their transitions
    int32_t G = 1;
    int64_t epoch = 0, adam_t = 0;
    uavrl::ReplayStore replay;        // int32 actions
    uavrl::LaunchChain chain;         // programmatic dependent launch state of the learner's stream (launch_chain.cuh)
    // prioritised replay (per.cuh); off unless uavrl_per_enable was called
    uavrl::PerDev per = {};
    uint64_t per_calls = 0;
    uint64_t act_calls = 0;
    uint64_t fed_calls = 0;           // ring-sampled federation calls: the Philox counter of their probe draws (federate.cu)
    // data-parallel: one-shot NVLink all-reduce fused with Adam (symmetric buffers exchanged through CUDA IPC), slots of P + 1
    // words (gradient, loss share)
    uavrl::PeerComm comm;
    unsigned long long *dp_trace = nullptr;    // UAVRL_DP_TRACE=1: phase times of the data-parallel optimiser kernel
    // owners of the buffers above, one per group allocated and replaced together: parameters, images, maps and dp_trace; the
    // grown scratch (partials, y / astar, act / dz rows); the PER trees; their scratch
    uavrl::DevMem mem, parts_mem, td_mem, rows_mem, per_mem, per_scratch_mem;
};

namespace uavrl {

// optimiser kernel arguments (reduce_adam_kernel, learner.cu; also launched by sac.cu)
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

// One exchange of dp_allreduce_adam_kernel (learner.cu): the optimiser steps of n_seg networks, segment k taking `blocks`
// blocks of 64 parameters after segment k - 1's and words [sum of the earlier P, + P) of a rank's slot, then n_extra scalar
// words: column j of the [n_extra_parts][extra_stride] partials, reduced by warp_column_sum and scaled, summed over ranks into
// extra_out[j].  Every rank's slot holds the words in that order.
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
// the exchange x on comm (its tag advances by one) with the Adam hyper-parameters of a; trace (may be null): UAVRL_DP_TRACE
cudaError_t launch_dp_exchange(PeerComm &comm, const AdamArgs &a, const DpExchange &x, cudaStream_t st, bool pdl,
                               unsigned long long *trace);

// reduce_adam_kernel (learner.cu) on `grid` (y: trainer) with the pointers of q; pdl: programmatic dependent launch
cudaError_t launch_reduce_adam(dim3 grid, cudaStream_t st, bool pdl, const AdamArgs &a, const AdamPtrs &q);

// torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8) at step t with learning rate lr: the fields of AdamArgs the step computes in
// double precision on the host (bias corrections, step size)
void adam_hyper(AdamArgs &a, float lr, int64_t t);
// every vector and image of a learner's optimiser step (trainer 0; the kernels offset by trainer)
AdamPtrs learner_adam_ptrs(const uavrl_learner *l, float *loss_out);

// Which kernels a pass over n rows per trainer takes on this learner, with its current switches (uavrl_learner_tc_route reports
// it): the act / TD pass and the update's training kernel each run on the tensor cores (generic or FIXED variant) or not.
struct Route {
    int fwd, train;               // tensor-core act / TD pass, training kernel: 0 = not used (fp32 kernel), 1 = generic, 2 = FIXED
    int fwd_rows, train_rows;     // their rows per tile (0 when not used)
    bool td_fused;                // the TD-target pass(es) run inside the training kernel
    bool fp32_dual;               // the fp32 update kernel keeps both networks' weights in shared memory at once
};
Route learner_route(const uavrl_learner *l, int n);

// The refusals both trainer-group create entry points make (uavrl_learner_create_trainers, uavrl_sac_create_trainers) after the
// learner's own configuration checks and before anything is allocated; on success cfg.device is current.  `learner` names the
// handle in the no-device message.
template <class Config>
int check_trainer_group(const Config &cfg, int32_t n_trainers, const char *learner)
{
    if (n_trainers < 1 || n_trainers > 65535)        // every grouped kernel runs one grid row per trainer: gridDim.y <= 65535
        return fail(UAVRL_ERR_INVALID, "n_trainers must be in [1, 65535]");
    if (n_trainers > 1 && (cfg.lockstep_envs < 0 || cfg.lockstep_envs % n_trainers != 0))
        return fail(UAVRL_ERR_INVALID, "lockstep_envs must be a multiple of n_trainers (every trainer owns lockstep_envs / n_trainers envs)");
    if (n_trainers > 1 && cfg.replay_capacity / n_trainers <= 0)
        return fail(UAVRL_ERR_INVALID, "replay_capacity / n_trainers must be > 0");
    if (cfg.batch_size <= 0 || cfg.replay_capacity <= 0) return fail(UAVRL_ERR_INVALID, "batch_size and replay_capacity must be > 0");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(UAVRL_ERR_CUDA, std::string("no CUDA device: the ") + learner + " has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg.device));
    return 0;
}

// Gradient / loss partial slots per trainer: a single trainer keeps max_ctas (any batch); a grouped learner sizes them from its
// per-trainer batch (the grid of its widest update kernel) and grows them when a larger explicit batch arrives.
inline int32_t trainer_parts_cap(int32_t G, int32_t batch_size, int32_t max_ctas)
{
    const int32_t tiles = (batch_size + kTile - 1) / kTile;
    return (G == 1 || tiles > max_ctas) ? max_ctas : tiles;
}

// generic MLP description: trunk widths + head = `head_main` rows (+ `head_extra` rows from a second parameter block)
int build_mlp(int in_dim, int n_hidden, const int32_t *hidden, int head_main, int head_extra, NetDev &n);
int launch_act(uavrl_learner *l, const float *obs, int n, float eps, int is_train, const float *u_tape,
               const int32_t *rand_tape, int32_t *actions, float *q_out, cudaStream_t st);
// the loss variant of the act pass (federation): weight sets w0 .. w0 + n_weights - 1 on the probe rows [G][kFedProbes][in_dim]
// (tc_forward.cuh TcArgs::loss_* for the row ranges), losses into loss_out[G][G]
int launch_fed_loss(uavrl_learner *l, const float *probes, const float *q_ref, float *loss_out, int w0, int n_weights, bool tri,
                    cudaStream_t st);
// One Trainer.update of B transitions per trainer (global_batch: the batch the loss averages over): gradient step, reduce (+ Adam
// when apply) into loss_out ([G]), prioritised-replay write-back.  marks (profiling, may be null): events recorded after the
// TD-target pass, the training kernel and the weight-gradient kernel; they change no launch.
int launch_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, bool apply, cudaStream_t st,
                  cudaEvent_t *marks = nullptr);
// the data-parallel form: the gradient step, then the NVLink all-reduce fused with Adam
int launch_update_dp(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, cudaStream_t st);
// the lockstep ring's commit plus, with prioritised replay, the priorities of the frames it makes and drops sampleable
void lockstep_commit(uavrl_learner *l, cudaStream_t st = nullptr);
}  // namespace uavrl
