// learner.cuh -- Q-network / replay / optimiser state of one learner (device-resident) + host handle.
#pragma once
#include "common.cuh"
#include "per.cuh"

namespace uavrl {

constexpr int kTile = 32;             // samples per CTA tile
constexpr int kNetThreads = 256;      // 8 warps: lane -> output unit, warp -> 4 samples
constexpr int kMaxDim = 128;          // every layer width (and in_dim) <= 128
constexpr int kMaxLayers = UAVRL_MAX_HIDDEN + 1;   // trunk layers + (combined) head

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

enum ReplayMode { kReplayPaired = 0, kReplayLockstep = 1, kBatchExplicit = 2 };

// where the rows of a batch come from
struct BatchSrc {
    int32_t mode;
    const float *frames;              // replay observation rows [rows][in_dim]
    const int32_t *act;               // [slots] discrete action index (DQN family)
    const float *act2;                // [slots][2] continuous action (SAC); nullptr otherwise
    const float *rew;                 // [slots]
    const uint8_t *done_u8;           // [slots]  (replay)          } one of the two
    const float *done_f32;            // [B]      (explicit batch)  }
    const float *s2_rows;             // explicit: next-state rows [B][in]
    const int32_t *idx_tape;          // optional injected indices [B]: logical (k-th oldest), or physical slots if idx_is_slot
    int32_t idx_is_slot;
    const float *is_w;                // optional per-sample importance weights (prioritised replay): loss = mean(w (Q-y)^2)
    float *abs_err;                   // optional out: |Q - y| per sample (ReplayTree.batch_update input)
    int64_t count, oldest;            // valid transitions, logical index of the oldest
    int64_t cap;                      // paired: slots ; lockstep: frames in the ring
    int32_t n_envs;                   // lockstep only: envs one trainer samples (count = frames x n_envs)
    int32_t row_stride;               // lockstep only: envs per ring frame (0 = n_envs); > n_envs for a grouped learner
    int32_t env_base;                 // lockstep only: first env sampled (trainer_src sets g x n_envs)
    uint64_t key, epoch;              // Philox key / counter for sampling
};

// Philox key salts of a learner seeded with `seed`: the eps-greedy draws use seed ^ kActSalt, replay sampling seed ^ kSampleSalt.
// Trainer g of a grouped learner draws exactly what a stand-alone learner seeded with seed + g draws.
constexpr uint64_t kActSalt = 0xAC7ull, kSampleSalt = 0x5EEDull;
__host__ __device__ __forceinline__ uint64_t trainer_key(uint64_t key, uint64_t salt, int g) { return ((key ^ salt) + (uint64_t)g) ^ salt; }

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
    // replay
    int32_t mode = 0;
    float *frames = nullptr;
    int32_t *r_act = nullptr;
    float *r_rew = nullptr;
    uint8_t *r_done = nullptr;
    int64_t slots = 0;                // paired: capacity ; lockstep: (ring_frames)*N
    int64_t ring_frames = 0;          // lockstep: frames in the ring (= capacity_frames + 1)
    int64_t head = 0;                 // paired: next slot to write ; lockstep: frame holding obs_t
    int64_t count = 0;                // valid transitions
    bool frame0_valid = false;
    // programmatic dependent launch chain of the lockstep loops (common.cuh)
    bool fuse_ok = false;             // the fused get_action + step kernel fits (tc_forward.cu)
    bool pdl_chain = false;
    int pdl_prev = 0;
    // prioritised replay (per.cuh); off unless uavrl_per_enable was called
    uavrl::PerDev per = {};
    uint64_t per_calls = 0;
    uint64_t act_calls = 0;
    // data-parallel: one-shot NVLink all-reduce fused with Adam (symmetric buffers exchanged through CUDA IPC)
    int32_t rank = 0, world = 1;
    float *comm_grad = nullptr;       // own receive buffer recv[2][world][P+1]: slot q is written by rank q (remote stores)
    int32_t comm_world = 0, comm_flag_words = 0;
    unsigned long long *dp_trace = nullptr;    // UAVRL_DP_TRACE=1: phase times of the data-parallel optimiser kernel
    unsigned *comm_flags = nullptr;   // own, [64]: slot q is raised by rank q
    unsigned *comm_counter = nullptr; // last-block detection of the publish kernel
    float **peer_grad_dev = nullptr;  // device array [world]: every rank's receive buffer as mapped on THIS device
    unsigned **peer_flag_dev = nullptr;
    void *peer_grad_host[64] = { nullptr }, *peer_flag_host[64] = { nullptr };
    bool comm_ready = false;
    unsigned flag_epoch = 0;
    unsigned long long *dw_bar = nullptr;      // fused weight-gradient + optimiser kernel: {epoch : value} partials [slices][P]
    unsigned long long dw_bar_total = 0;
    int last_nparts = 0, last_n_loss_parts = 0;
    int last_global_batch = 0;
};

namespace uavrl {

#if defined(__CUDACC__)
__device__ __forceinline__ uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}

// i-th element of a keyed pseudo-random permutation of [0, M): 4-round Feistel on 2*h bits with
// cycle walking.  perm(0..B-1) = B distinct uniform indices = random.sample(range(M), B)
// (BaseClass/replay_buffer.py:49).
__device__ __forceinline__ uint64_t perm_index(uint64_t i, uint64_t M, const uint32_t key[4])
{
    int bits = 1;
    while ((1ull << bits) < M) ++bits;
    const int h = (bits + 1) / 2;
    const uint32_t mask = (h >= 32) ? 0xffffffffu : ((1u << h) - 1u);
    uint64_t x = i;
    do {
        uint32_t Lh = (uint32_t)(x >> h) & mask, Rh = (uint32_t)x & mask;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const uint32_t f = mix32(Rh ^ key[r]) & mask;
            const uint32_t nl = Rh;
            Rh = Lh ^ f;
            Lh = nl;
        }
        x = ((uint64_t)Lh << h) | Rh;
    } while (x >= M);
    return x;
}

// batch position gb -> the transition's state row, next-state row and metadata
struct Transition { const float *s, *s2; int a; float r, d, ax, ay; };
// the two halves of resolve_transition: (1) where the rows are -- index arithmetic only, nothing a predecessor kernel writes is
// read (an index tape, when present, comes from a kernel that is never a programmatic-launch predecessor); (2) the
// transition's action / reward / done, which the env step of the same iteration may just have written
// fresh: the next-state row lies in the frame the env step of the SAME iteration writes (lockstep ring: the frame behind the
// newest transition group) -- the only sampled row a kernel launched programmatically behind that env step must not read early
// Trainer g's view of a batch source (grouped learner: gridDim.y = G trainers, B rows each).  Explicit batches: block g of the
// G x B rows.  Lockstep ring: env block [g n_envs, (g + 1) n_envs), trainer g's sampling key and row g of a [G][B] index tape.
__device__ __forceinline__ BatchSrc trainer_src(BatchSrc s, int g, int B, int in_dim)
{
    if (g == 0) return s;
    const size_t r0 = (size_t)g * (size_t)B;
    if (s.mode == kBatchExplicit) {
        s.frames += r0 * in_dim; s.s2_rows += r0 * in_dim; s.rew += r0; s.done_f32 += r0;
        if (s.act) s.act += r0;
        if (s.act2) s.act2 += 2 * r0;
        return s;
    }
    s.env_base = g * s.n_envs;
    s.key = trainer_key(s.key, kSampleSalt, g);
    if (s.idx_tape) s.idx_tape += r0;
    return s;
}

__device__ __forceinline__ int64_t resolve_rows(const BatchSrc &src, int gb, int in_dim, const uint32_t pkey[4], const float *&s, const float *&s2,
                                                bool *fresh = nullptr)
{
    if (fresh) *fresh = false;
    if (src.mode == kBatchExplicit) {
        s = src.frames + (size_t)gb * in_dim; s2 = src.s2_rows + (size_t)gb * in_dim;
        return gb;
    }
    const uint64_t j = src.idx_tape ? (uint64_t)src.idx_tape[gb] : perm_index((uint64_t)gb, (uint64_t)src.count, pkey);
    int64_t slot, row, row2;
    if (src.mode == kReplayLockstep) {
        const int64_t N = src.row_stride ? src.row_stride : src.n_envs;
        const int64_t f = src.idx_is_slot ? (int64_t)(j / src.n_envs) : (src.oldest + (int64_t)(j / src.n_envs)) % src.cap;
        const int64_t e = src.env_base + (int64_t)(j % src.n_envs);
        slot = f * N + e; row = slot;
        row2 = ((f + 1) % src.cap) * N + e;
        if (fresh) *fresh = ((f + 1) % src.cap) == (src.oldest + src.count / src.n_envs) % src.cap;
    } else {
        slot = src.idx_is_slot ? (int64_t)j : (src.oldest + (int64_t)j) % src.cap; row = 2 * slot; row2 = 2 * slot + 1;
    }
    s = src.frames + (size_t)row * in_dim; s2 = src.frames + (size_t)row2 * in_dim;
    return slot;
}
__device__ __forceinline__ void load_meta(const BatchSrc &src, int64_t slot, int &a, float &r, float &d)
{
    a = src.act ? src.act[slot] : 0; r = src.rew[slot];
    d = (src.mode == kBatchExplicit) ? src.done_f32[slot] : (src.done_u8[slot] ? 1.f : 0.f);
}
__device__ __forceinline__ Transition resolve_transition(const BatchSrc &src, int gb, int in_dim, const uint32_t pkey[4])
{
    Transition t;
    if (src.mode == kBatchExplicit) {
        t.s = src.frames + (size_t)gb * in_dim;
        t.s2 = src.s2_rows + (size_t)gb * in_dim;
        t.a = src.act ? src.act[gb] : 0; t.r = src.rew[gb]; t.d = src.done_f32[gb];
        t.ax = src.act2 ? src.act2[2 * gb] : 0.f; t.ay = src.act2 ? src.act2[2 * gb + 1] : 0.f;
        return t;
    }
    const uint64_t j = src.idx_tape ? (uint64_t)src.idx_tape[gb] : perm_index((uint64_t)gb, (uint64_t)src.count, pkey);
    int64_t slot, row, row2;
    if (src.mode == kReplayLockstep) {
        const int64_t N = src.row_stride ? src.row_stride : src.n_envs;
        const int64_t f = src.idx_is_slot ? (int64_t)(j / src.n_envs) : (src.oldest + (int64_t)(j / src.n_envs)) % src.cap;
        const int64_t e = src.env_base + (int64_t)(j % src.n_envs);
        slot = f * N + e; row = slot;
        row2 = ((f + 1) % src.cap) * N + e;
    } else {
        slot = src.idx_is_slot ? (int64_t)j : (src.oldest + (int64_t)j) % src.cap; row = 2 * slot; row2 = 2 * slot + 1;
    }
    t.s = src.frames + (size_t)row * in_dim;
    t.s2 = src.frames + (size_t)row2 * in_dim;
    t.a = src.act ? src.act[slot] : 0; t.r = src.rew[slot]; t.d = src.done_u8[slot] ? 1.f : 0.f;
    t.ax = src.act2 ? src.act2[2 * slot] : 0.f; t.ay = src.act2 ? src.act2[2 * slot + 1] : 0.f;
    return t;
}
#endif

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
    // every operation individually rounded (no FMA contraction): the optimiser kernels that share this function (stand-alone,
    // fused behind the weight-gradient kernel, all-reduce) then produce bit-identical parameters by construction
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

__device__ __forceinline__ void adam_update_one(const AdamArgs &a, const AdamPtrs &q, int i, float g)
{
    adam_update_pre(a, q, i, g, adam_prefetch(q, i));
}

__global__ void reduce_adam_kernel(AdamArgs a, const float *__restrict__ partials, const float *__restrict__ loss_partials,
                                   float *__restrict__ grad, float *__restrict__ local, float *__restrict__ m, float *__restrict__ v,
                                   float *__restrict__ target, float *__restrict__ img_local, float *__restrict__ img_target,
                                   const int32_t *__restrict__ img_map, float *__restrict__ tc_local, float *__restrict__ tc_target,
                                   const int32_t *__restrict__ tc_hi, const int32_t *__restrict__ tc_lo, const int32_t *__restrict__ tc_hi2,
                                   const int32_t *__restrict__ tc_lo2, float *__restrict__ loss_out);
#endif

// generic MLP description: trunk widths + head = `head_main` rows (+ `head_extra` rows from a second parameter block)
int build_mlp(int in_dim, int n_hidden, const int32_t *hidden, int head_main, int head_extra, NetDev &n);
struct EnvDev;
extern std::atomic<int> g_fuse_act_env;
int launch_act_env(uavrl_learner *l, const EnvDev &d, const float *obs, float eps, int32_t *actions, float *obs_next, float *rew,
                   uint8_t *done, cudaStream_t st);
int launch_act(uavrl_learner *l, const float *obs, int n, float eps, int is_train, const float *u_tape,
               const int32_t *rand_tape, int32_t *actions, float *q_out, cudaStream_t st);
int launch_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out,
                  bool apply, cudaStream_t st);
int launch_update_dp(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, cudaStream_t st);
int launch_update_split(uavrl_learner *l, const BatchSrc &src, int B, cudaStream_t st, cudaEvent_t *mid);
int lockstep_begin(uavrl_learner *l, float **obs_t, float **obs_next, int32_t **act, float **rew, uint8_t **done);
void lockstep_commit(uavrl_learner *l, cudaStream_t st = nullptr);
BatchSrc replay_source(uavrl_learner *l, const int32_t *idx_tape);
}  // namespace uavrl
