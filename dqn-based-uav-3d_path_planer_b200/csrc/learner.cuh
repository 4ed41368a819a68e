// learner.cuh -- Q-network / replay / optimiser state of one learner (device-resident) + host handle.
#pragma once
#include "net.cuh"
#include "optim.cuh"
#include "replay.cuh"

namespace uavrl {

constexpr int kFedProbes = 10;        // probe states per trainer of a federation round (PathPlan_City.py:658)

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

// Federation: the loss entry of one probe group, loss_out[p * ld + col] = (sum of its kFedProbes rows' squared Q differences
// d2, in row order) / (S A); first_row = the group's first row in the [G][S] probe rows, p = its trainer.
__device__ __forceinline__ void fed_group_loss(const float *d2, size_t first_row, int ld, int col, int n_actions, float *loss_out)
{
    float s2 = 0.f;
    for (int r = 0; r < kFedProbes; ++r) s2 += d2[r];
    const size_t p = first_row / kFedProbes;
    loss_out[p * (size_t)ld + col] = s2 / (float)(kFedProbes * n_actions);
}
#endif

// The sharded federation (federate.cu, uavrl_learner_fed_shard): this learner's G_local trainers are the global trainers
// [rank G_local, (rank + 1) G_local) of G = G_local world.  Two buffers are exchanged by all-gathers in rank order:
//   x0 [G][S in + S A + P]: every trainer's [probes | q_ref | q_local] (phase 0);
//   x1 [world][G][G_local]: every rank's columns of the initial loss matrix (phase 1).
// The rest is scratch of the rounds: the gathered rows unpacked into probes [G][S][in], q_ref [G][S][A] and the flat replica
// rep [G][P] of every q_local, the loss matrix M [G][G], the chosen lists [G][max(1, k)], the weight images (fp32 and tensor
// core) of the trainer a round has just averaged, and the local phase's probe rows, Q rows and actions.
struct FedShard {
    int32_t rank = 0, world = 0;              // world 0: no shard declared
    int32_t phase = 0;                        // 0: ready for the local phase, 1: x0 slice written, 2: x1 slice written
    float *x0 = nullptr, *x1 = nullptr;
    float *probes = nullptr, *q_ref = nullptr, *rep = nullptr, *M = nullptr, *img = nullptr;
    unsigned char *tc_img = nullptr;
    float *l_probes = nullptr, *l_q = nullptr;
    int32_t *chosen = nullptr, *acts = nullptr;
    DevMem mem;
};

// One loss pass of the federation (launch_fed_loss) over the probe rows [G][kFedProbes][in_dim] of G trainers and their reference
// Q rows [G][kFedProbes][A]: weight set w evaluates image w - img0 of img (fp32 route) or tc_img (tensor-core route) and writes
// loss_out[p * ld + w - col0] for every probe group p it covers.
struct FedLoss {
    const float *probes, *q_ref;
    float *loss_out;
    int G, ld, col0, img0;
    const float *img;
    const unsigned char *tc_img;
};

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
    uavrl::ReplayStore replay;        // int32 actions; with prioritised replay, its SumTrees
    uavrl::LaunchChain chain;         // programmatic dependent launch state of the learner's stream (launch_chain.cuh)
    uint64_t act_calls = 0;
    uint64_t fed_calls = 0;           // ring-sampled federation calls: the Philox counter of their probe draws (federate.cu)
    uavrl::FedShard fed;              // the sharded federation's rank, phase and buffers
    // data-parallel: one-shot NVLink all-reduce fused with Adam (symmetric buffers exchanged through CUDA IPC), slots of P + 1
    // words (gradient, loss share)
    uavrl::PeerComm comm;
    // owners of the buffers above, one per group allocated and replaced together: parameters, images, maps; the
    // grown scratch (partials, y / astar, act / dz rows)
    uavrl::DevMem mem, parts_mem, td_mem, rows_mem;
};

namespace uavrl {
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

int launch_act(uavrl_learner *l, const float *obs, int n, float eps, int is_train, const float *u_tape,
               const int32_t *rand_tape, int32_t *actions, float *q_out, cudaStream_t st);
// the loss variant of the act pass (federation): weight sets w0 .. w0 + n_weights - 1 on the probe rows of f (tc_forward.cuh
// TcArgs::loss_* for the row ranges).  The route follows from f.G alone, so every entry is the same sum whichever launch makes it.
int launch_fed_loss(uavrl_learner *l, const FedLoss &f, int w0, int n_weights, bool tri, cudaStream_t st);
// One Trainer.update of B transitions per trainer (global_batch: the batch the loss averages over): gradient step, reduce (+ Adam
// when apply) into loss_out ([G]), prioritised-replay write-back.  marks (profiling, may be null): events recorded after the
// TD-target pass, the training kernel and the weight-gradient kernel; they change no launch.
int launch_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, bool apply, cudaStream_t st,
                  cudaEvent_t *marks = nullptr);
// the data-parallel form: the gradient step, then the NVLink all-reduce fused with Adam
int launch_update_dp(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, cudaStream_t st);
}  // namespace uavrl
