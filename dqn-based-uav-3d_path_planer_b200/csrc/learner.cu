// learner.cu -- DQN-family learner on device: Q-net forward + eps-greedy, replay ring, sampled
// TD update (forward local/target, MSE, backward), Adam, hard target update.  sm_90a.
//
// Replaces (SURVEY.md section 8a rows a-10..a-13):
//   Trainer.get_action        Trainer/DuelingDQN_Trainer.py:86-97
//   ReplayMemory.add/sample2  BaseClass/replay_buffer.py:41-51
//   Trainer.update            Trainer/DuelingDQN_Trainer.py:150-190, Trainer/DDQN_Trainer.py:72-117,
//                             Trainer/DQN_Trainer.py:85-136
//   networks                  BaseClass/BaseCNN.py:93-102,120-217,329-343
//   torch.optim.Adam step + hard_update (DuelingDQN_Trainer.py:176-184,199-202): launched here, kernels in optim.cu
//
// This file is the fp32 CUDA-core path: the whole network (<= 23 k parameters) is staged TRANSPOSED in
// shared memory once per CTA, a CTA owns a tile of 32 samples, lanes walk output units and each
// warp carries 4 samples, so every weight fetch is a conflict-free LDS and every activation fetch
// a broadcast LDS.128.  Gradients leave the CTA as one coalesced partial vector; the optimiser
// kernel (optim.cu) reduces the partials in a fixed order (deterministic) and applies Adam.
#include "learner.cuh"
#include "mlp_tile.cuh"
#include "tc_forward.cuh"

#include <math.h>
#include <string.h>

#include <string>
#include <vector>

namespace uavrl {

// ------------------------------------------------------------------ network description (host)
static int build_net(const uavrl_learner_config &c, NetDev &n)
{
    if (c.n_actions < 1 || c.n_actions > 31) return fail(UAVRL_ERR_INVALID, "n_actions must be in [1,31]");
    int rc = build_mlp(c.in_dim, c.n_hidden, c.hidden, c.n_actions, c.dueling ? 1 : 0, n);
    if (rc) return rc;
    n.dueling = c.dueling ? 1 : 0;
    return 0;
}

// ------------------------------------------------------------------ eps-greedy action kernel
// LOSS (federation, launch_fed_loss): grid row y evaluates weight set w = fl.w0 + y on probe rows [0, S w) (fl.tri) or
// [S (w + 1), n) of obs = [G][S][in_dim], S = kFedProbes, with image w - fl.img0; a tile takes 3 whole probe groups (30 rows)
// and writes fl.loss_out[p * fl.ld + w - fl.col0] = sum over trainer p's rows of sum_a (fl.q_ref - Q_w)^2 / (S A).  The same
// reduction as the tensor-core loss variant (tc_forward.cu).
struct FedLossArgs { const float *q_ref; float *loss_out; int w0, tri, img0, ld, col0; };

template <bool LOSS>
__global__ void __launch_bounds__(kNetThreads)
act_kernel_t(NetDev net, const float *__restrict__ params, const float *__restrict__ obs, int n, float eps,
             int is_train, const float *__restrict__ u_tape, const int32_t *__restrict__ rand_tape,
             uint64_t key, uint64_t call, int32_t *__restrict__ actions, int32_t *__restrict__ actions2,
             float *__restrict__ q_out, int n_tiles, int img_floats, FedLossArgs fl)
{
    extern __shared__ __align__(16) float smem[];
    constexpr int kStep = LOSS ? (kTile / kFedProbes) * kFedProbes : kTile;      // rows a tile advances by
    int w_set = 0, n_rows = n;
    size_t row0 = 0;
    if (LOSS) {
        w_set = fl.w0 + blockIdx.y;
        const int lo = fl.tri ? 0 : kFedProbes * (w_set + 1), hi = fl.tri ? kFedProbes * w_set : n;
        row0 = (size_t)lo; n_rows = hi - lo;
        n_tiles = (n_rows + kStep - 1) / kStep;
        if ((int)blockIdx.x >= n_tiles) return;
        params += (size_t)(w_set - fl.img0) * img_floats; obs += row0 * net.in_dim;
    } else {   // trainer blockIdx.y of a grouped learner: its weight image, its n rows and its eps-greedy key
        const int g = blockIdx.y;
        const size_t r0 = (size_t)g * (size_t)n;
        params += (size_t)g * img_floats; obs += r0 * net.in_dim; actions += r0;
        if (actions2) actions2 += r0;
        if (q_out) q_out += r0 * net.n_actions;
        if (u_tape) u_tape += r0;
        if (rand_tape) rand_tape += r0;
        key = trainer_key(key, kActSalt, g);
    }
    float *sw = smem;
    float *sA = smem + net.smem_total_floats;
    float *sB = sA + kTile * kMaxDim;
    float *head = sB + kTile * kMaxDim;
    __shared__ const float *rows[kTile];
    __shared__ uint64_t wbar;
    if (threadIdx.x == 0) { mbar_init(&wbar, 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) stage_weights(net, params, sw, &wbar);      // params = the network's smem image
    bool weights_ready = false;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int e0 = t * kStep;
        if (threadIdx.x < kTile)
            rows[threadIdx.x] = (threadIdx.x < kStep && e0 + threadIdx.x < n_rows) ? obs + (size_t)(e0 + threadIdx.x) * net.in_dim : nullptr;
        __syncthreads();
        if (net.in_dim % 4 == 0) load_rows(rows, smem + net.act_off[0], net.act_ld[0], net.in_dim);
        else load_rows_scalar(rows, smem + net.act_off[0], net.act_ld[0], net.in_dim);
        if (!weights_ready) { mbar_wait(&wbar, 0); weights_ready = true; }
        __syncthreads();
        net_forward(net, sw, smem + net.act_off[0], net.act_ld[0], smem, false, sA, sB, head);
        if (LOSS) {
            if (threadIdx.x < kTile) {
                float d2 = 0.f;
                if (threadIdx.x < kStep && e0 + threadIdx.x < n_rows) {
                    const float *row = head + threadIdx.x * 32, *ref = fl.q_ref + (row0 + e0 + threadIdx.x) * net.n_actions;
                    for (int k = 0; k < net.n_actions; ++k) { const float d = ref[k] - row[k]; d2 += d * d; }
                }
                sA[threadIdx.x] = d2;                     // sA: free scratch once the forward is done
            }
            __syncthreads();
            if (threadIdx.x * kFedProbes < kStep && e0 + (int)threadIdx.x * kFedProbes < n_rows)
                fed_group_loss(sA + threadIdx.x * kFedProbes, row0 + e0 + threadIdx.x * kFedProbes, fl.ld, w_set - fl.col0, net.n_actions, fl.loss_out);
        } else if (threadIdx.x < kTile && e0 + threadIdx.x < n) {
            const int e = e0 + threadIdx.x;
            const float *row = head + threadIdx.x * 32;
            int ra;
            const int a = eps_greedy(eps, is_train, u_tape, rand_tape, e, key, call, e, net.n_actions, ra) ? argmax_row(row, net.n_actions) : ra;
            actions[e] = a;
            if (actions2) actions2[e] = a;
            if (q_out) for (int k = 0; k < net.n_actions; ++k) q_out[(size_t)e * net.n_actions + k] = row[k];
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ TD update kernel
struct UpdateArgs {
    const float *img_local, *img_target;
    float *partials, *loss_partials;
    int B, n_tiles, algo, dual, loss_kind;
    int img_floats;                    // grouped learner: per-trainer stride of the weight images
    float gamma, inv_global_b;
    const float *y_in;                 // non-null: TD targets already computed (tensor-core pass); skip the target net
};

// smem: [W primary (local)] [W secondary (target), only if dual] [planes X0,H1..] [X2] [sA] [sB] [Q] [Qt] [Ql2]
__global__ void __launch_bounds__(kNetThreads)
update_kernel(NetDev net, BatchSrc src, UpdateArgs ua)
{
    extern __shared__ __align__(16) float smem[];
    const int wf = net.smem_w_floats;
    float *swL = smem;                                   // local image (single-buffer mode: whichever net is live)
    float *swT = ua.dual ? smem + wf : smem;
    float *pl = smem + (ua.dual ? wf : 0);               // base the NetDev plane offsets are relative to
    float *X0 = pl + net.act_off[0];
    const int ld0 = net.act_ld[0];
    float *X2 = pl + net.smem_total_floats;              // next-state plane
    float *sA = X2 + kTile * ld0;                        // scratch / gradient ping
    float *sB = sA + kTile * kMaxDim;                    // scratch / gradient pong
    float *Q = sB + kTile * kMaxDim;                     // [32][32] Q_local(s)
    float *Qt = Q + kTile * 32;                          // [32][32] Q_target(s')
    float *Ql2 = Qt + kTile * 32;                        // [32][32] Q_local(s')
    __shared__ const float *rows_s[kTile];
    __shared__ const float *rows_s2[kTile];
    __shared__ int s_act[kTile];
    __shared__ float s_rew[kTile], s_done[kTile], s_loss[kTile];
    __shared__ uint64_t barL, barT;

    // trainer blockIdx.y of a grouped learner: its B samples, weight images and partial slots [G][gridDim.x]
    const int grp = blockIdx.y;
    src = trainer_src(src, grp, ua.B, net.in_dim);
    {
        const size_t wo = (size_t)grp * ua.img_floats;
        ua.img_local += wo; ua.img_target += wo;
        if (ua.y_in) ua.y_in += (size_t)grp * ua.B;
    }
    const size_t part = (size_t)grp * gridDim.x + blockIdx.x;
    float *gpart = ua.partials + part * net.P;
    float loss_acc = 0.f;
    int iter = 0;
    uint32_t pkey[4];
    Philox::gen(src.key, src.epoch, 0x5A17ull, pkey);
    uint32_t phL = 0, phT = 0;

    if (threadIdx.x == 0) { mbar_init(&barL, 1); mbar_init(&barT, 1); fence_barrier_init(); }
    __syncthreads();
    const bool have_y = ua.y_in != nullptr;
    if (threadIdx.x == 0) {
        if (have_y) stage_weights(net, ua.img_local, swL, &barL);       // only the local network is evaluated here
        else {
            stage_weights(net, ua.img_target, swT, &barT);              // target first: it is needed first
            if (ua.dual) stage_weights(net, ua.img_local, swL, &barL);
        }
    }

    for (int t = blockIdx.x; t < ua.n_tiles; t += gridDim.x, ++iter) {
        // ---- resolve the tile's transitions
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr; tr.s2 = nullptr; tr.a = 0; tr.r = 0.f; tr.d = 0.f;
            if (gb < ua.B) tr = resolve_transition(src, gb, net.in_dim, pkey);
            rows_s[threadIdx.x] = tr.s; rows_s2[threadIdx.x] = ua.y_in ? nullptr : tr.s2;
            s_act[threadIdx.x] = tr.a; s_rew[threadIdx.x] = tr.r; s_done[threadIdx.x] = tr.d;
        }
        __syncthreads();
        if (net.in_dim % 4 == 0) { load_rows(rows_s, X0, ld0, net.in_dim); if (!have_y) load_rows(rows_s2, X2, ld0, net.in_dim); }
        else { load_rows_scalar(rows_s, X0, ld0, net.in_dim); if (!have_y) load_rows_scalar(rows_s2, X2, ld0, net.in_dim); }
        if (have_y) {
            if (iter == 0) { mbar_wait(&barL, phL); phL ^= 1; }
            __syncthreads();
        } else {
            // ---- target network on s'
            if (!ua.dual && iter > 0) {                   // single buffer: bring the target image back
                __syncthreads();
                if (threadIdx.x == 0) stage_weights(net, ua.img_target, swT, &barT);
            }
            if (!ua.dual || iter == 0) { mbar_wait(&barT, phT); phT ^= 1; }
            __syncthreads();
            net_forward(net, swT, X2, ld0, pl, false, sA, sB, Qt);
            // ---- local network on s' (double-DQN action selection)
            if (!ua.dual) {
                if (threadIdx.x == 0) stage_weights(net, ua.img_local, swL, &barL);
                mbar_wait(&barL, phL); phL ^= 1;
            } else if (iter == 0) { mbar_wait(&barL, phL); phL ^= 1; }
            __syncthreads();
            if (ua.algo != UAVRL_ALGO_DQN) net_forward(net, swL, X2, ld0, pl, false, sA, sB, Ql2);
        }
        // ---- local network on s (activations kept for backward)
        net_forward(net, swL, X0, ld0, pl, true, sA, sB, Q);
        // ---- TD target, loss, dLoss/dHead  (head gradient plane = sA, [32][kMaxDim], zero padded)
        const int nA = net.n_actions;
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x;
            float *g = sA + b * kMaxDim;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            float lossb = 0.f;
            if (t * kTile + b < ua.B) {
                float y;
                if (have_y) y = ua.y_in[t * kTile + b];
                else {
                    const float *qt = Qt + b * 32;
                    float nq;
                    if (ua.algo == UAVRL_ALGO_DQN) nq = qt[argmax_row(qt, nA)];       // DQN_Trainer.py:109
                    else nq = qt[argmax_row(Ql2 + b * 32, nA)];                      // DDQN_Trainer.py:94-95
                    y = td_target(s_rew[b], ua.gamma, nq, s_done[b]);
                }
                const int a = s_act[b];
                float gq;
                lossb = td_loss(src, t * kTile + b, Q[b * 32 + a] - y, ua.loss_kind, ua.inv_global_b, gq);
                if (net.dueling) {
                    const float inv = 1.f / (float)nA;
                    for (int o = 0; o < nA; ++o) g[o] = gq * ((o == a ? 1.f : 0.f) - inv);
                    g[nA] = gq;
                } else {
                    g[a] = gq;
                }
            }
            s_loss[b] = lossb;
        }
        __syncthreads();
        if (threadIdx.x == 0) { float s = 0.f; for (int b = 0; b < kTile; ++b) s += s_loss[b]; loss_acc += s; }
        // ---- backward, head first.  gradient planes ping-pong sA <-> sB
        float *dY = sA, *dXb = sB;
        for (int l = net.n_layers - 1; l >= 0; --l) {
            const LayerDev &L = net.L[l];
            const float *Xin = pl + net.act_off[l];
            const int ldx = net.act_ld[l];
            layer_backward_dw(dY, kMaxDim, Xin, ldx, gpart, L, iter > 0);
            if (l > 0) {
                layer_backward_dx(dY, kMaxDim, swL + L.smem_w, Xin, ldx, dXb, kMaxDim, L.in, L.out);
                // zero the pad columns [in, round_up(in,32)) the next dW pass will read
                const int pad0 = L.in, pad1 = round_up(L.in, 32);
                for (int i = threadIdx.x; i < kTile * (pad1 - pad0); i += blockDim.x)
                    dXb[(i / (pad1 - pad0)) * kMaxDim + pad0 + i % (pad1 - pad0)] = 0.f;
            }
            __syncthreads();
            float *tmp = dY; dY = dXb; dXb = tmp;
        }
    }
    if (threadIdx.x == 0) ua.loss_partials[part] = loss_acc;
}

__global__ void copy_kernel(size_t n, const float *__restrict__ src, float *__restrict__ dst)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
static void launch_copy(size_t n, const float *src, float *dst, cudaStream_t st)
{
    const size_t blocks = (n + 255) / 256;
    copy_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 256, 0, st>>>(n, src, dst);
}

// ------------------------------------------------------------------ host launchers
static size_t act_smem_bytes(const NetDev &n) { return (size_t)(n.smem_total_floats + 2 * kTile * kMaxDim + kTile * 32) * 4; }
static size_t upd_smem_bytes(const NetDev &n, int dual)
{
    return (size_t)((dual ? n.smem_w_floats : 0) + n.smem_total_floats + kTile * n.act_ld[0] + 2 * kTile * kMaxDim +
                    3 * kTile * 32) * 4;
}

std::atomic<int> g_fuse_td{1};               // uavrl_set_fuse_td(); default on

Route learner_route(const uavrl_learner *l, int n)
{
    Route r;
    memset(&r, 0, sizeof(r));
    r.fp32_dual = l->dual_weights != 0;
    if (!l->tc_ok || !l->use_tc) return r;
    const int n_sm = num_sms();
    r.fwd = l->tc_fixed_fwd ? 2 : 1;
    // act / TD pass: the largest tile of which the rows fill a wave (128 rows only when that image fits shared memory)
    r.fwd_rows = (n >= 128 * n_sm && l->tc.max_rows == 128) ? 128 : (n >= 64 * n_sm) ? 64 : 32;
    if (!l->tc_train_ok) return r;
    r.train = l->tc_fixed_train ? 2 : 1;
    // training kernel: 32 rows while the batch fits one wave of 32-row tiles, else 64 (when the 64-row operands fit)
    r.train_rows = (n > 32 * n_sm && l->tc.train_max_rows == 64) ? 64 : 32;
    // TD passes inside the training kernel at one tile per CTA (32-row tiles up to 4 736 samples, 64-row tiles up to 9 472): the
    // weight images are restaged inside the kernel, which only pays when a CTA does it once; larger batches keep the separate
    // TD-target kernel(s), whose CTAs reuse one image over several tiles
    r.td_fused = g_fuse_td.load() && (n + r.train_rows - 1) / r.train_rows <= n_sm;
    return r;
}

int launch_act(uavrl_learner *l, const float *obs, int n_all, float eps, int is_train, const float *u_tape,
               const int32_t *rand_tape, int32_t *actions, float *q_out, cudaStream_t st)
{
    const int n = n_all / l->G;                          // rows per trainer (grouped learner: G equal blocks)
    const Route r = learner_route(l, n);
    if (r.fwd) {                                         // tensor-core forward chain (tc_forward.cu)
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.img = l->tc_img_local; a.obs = obs; a.n = n; a.mode = kTcAct;
        a.eps = eps; a.is_train = is_train; a.u_tape = u_tape; a.rand_tape = rand_tape;
        a.key = l->cfg.seed ^ kActSalt; a.call = l->act_calls++; a.actions = actions; a.q_out = q_out;
        return launch_tc_forward(l, r, a, st);
    }
    const int n_tiles = (n + kTile - 1) / kTile;
    const int grid = n_tiles < 4 * num_sms() ? n_tiles : 4 * num_sms();
    act_kernel_t<false><<<dim3(grid, l->G), kNetThreads, act_smem_bytes(l->net), st>>>(l->net, l->img_local, obs, n, eps, is_train, u_tape,
                                                                                      rand_tape, l->cfg.seed ^ kActSalt, l->act_calls++,
                                                                                      actions, nullptr, q_out, n_tiles, l->net.smem_w_floats,
                                                                                      FedLossArgs{});
    l->chain.launched(kChainNone);
    UAVRL_LAUNCHED();
    return 0;
}

int launch_fed_loss(uavrl_learner *l, const FedLoss &f, int w0, int n_weights, bool tri, cudaStream_t st)
{
    const int n = f.G * kFedProbes;                      // every probe row; a weight set evaluates at most n - S of them
    const int max_rows = n - kFedProbes;
    if (max_rows <= 0 || n_weights <= 0) return 0;
    const Route r = learner_route(l, max_rows);
    if (r.fwd) {
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.img = f.tc_img; a.obs = f.probes; a.n = n; a.mode = kTcAct;
        a.q_ref = f.q_ref; a.loss_out = f.loss_out; a.loss_w0 = w0; a.loss_tri = tri ? 1 : 0;
        a.loss_img0 = f.img0; a.loss_ld = f.ld; a.loss_col0 = f.col0;
        return launch_tc_loss(l, r, a, n_weights, max_rows, st);
    }
    constexpr int step = (kTile / kFedProbes) * kFedProbes;
    const int n_tiles = (max_rows + step - 1) / step;
    const int grid = n_tiles < 4 * num_sms() ? n_tiles : 4 * num_sms();
    act_kernel_t<true><<<dim3(grid, n_weights), kNetThreads, act_smem_bytes(l->net), st>>>(l->net, f.img, f.probes, n, 0.f, 0, nullptr,
                                                                                          nullptr, 0, 0, nullptr, nullptr, nullptr, n_tiles,
                                                                                          l->net.smem_w_floats,
                                                                                          FedLossArgs{ f.q_ref, f.loss_out, w0, tri ? 1 : 0,
                                                                                                       f.img0, f.ld, f.col0 });
    l->chain.launched(kChainNone);
    UAVRL_LAUNCHED();
    return 0;
}

// ---- one Trainer.update: the gradient step (launch_grads), the optimiser step (adam_args and a launcher per kind), and the
// prioritised-replay write-back (per_write_back), always in that order

// what the gradient step leaves for the optimiser step
struct Grads {
    int rc;                       // != 0: the gradient step failed
    int nparts, n_loss_parts;     // gradient / loss partial slots written per trainer; 0: l->grad already holds the gradient
    float inv_b;                  // 1 / the batch the loss averages over
    bool per;                     // sampled from the SumTree: the |Q - y| of the batch go back to it
};

// the fp32 CUDA-core update kernel on `grid` CTAs per trainer: TD targets (unless y_in holds them), forward, backward and the
// weight-gradient partials in one launch
static int launch_fp32_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, int grid, const float *y_in,
                              cudaStream_t st)
{
    UpdateArgs ua;
    ua.img_local = l->img_local; ua.img_target = l->img_target; ua.partials = l->partials; ua.loss_partials = l->loss_partials;
    ua.B = B; ua.n_tiles = (B + kTile - 1) / kTile; ua.algo = l->cfg.algo; ua.gamma = l->cfg.gamma; ua.dual = l->dual_weights;
    ua.loss_kind = l->cfg.loss_kind; ua.img_floats = l->net.smem_w_floats;
    ua.inv_global_b = 1.0f / (float)global_batch;
    ua.y_in = y_in;
    update_kernel<<<dim3(grid, l->G), kNetThreads, upd_smem_bytes(l->net, l->dual_weights), st>>>(l->net, src, ua);
    l->chain.launched(kChainNone);
    UAVRL_LAUNCHED();
    return 0;
}

static int mark(cudaEvent_t *marks, int k, cudaStream_t st)
{
    if (marks) UAVRL_CUDA(cudaEventRecord(marks[k], st));
    return 0;
}

// Sample (prioritised replay), TD-target pass(es) and training kernel(s): the gradient partials of B transitions per trainer.
// marks (profiling, may be null): events after the TD-target pass, the training kernel and the weight-gradient kernel (the
// training kernel on the fp32 path, which computes the weight gradients itself)
static Grads launch_grads(uavrl_learner *l, const BatchSrc &src_in, int B, int global_batch, cudaStream_t st, cudaEvent_t *marks)
{
    Grads g = { 0, 0, 0, 1.0f / (float)global_batch, l->replay.per_samples(src_in) };
    BatchSrc src = src_in;
    if (g.per) {
        // ReplayTree.sample2 -> slots + importance weights; |Q - y| comes back for batch_update (per_write_back)
        src = l->replay.per_source(l->cfg.seed, B, src_in, st, &g.rc);
        if (g.rc) return g;
        l->chain.launched(kChainNone);                    // prioritised-replay kernels launch outside the chain
    }
    const Route r = learner_route(l, B);
    const int n_tiles = (B + kTile - 1) / kTile;
    const int grid = n_tiles < l->max_ctas ? n_tiles : l->max_ctas;
    if ((g.rc = grow(l->parts_mem, l->parts_cap, grid, st, true,      // grouped learner, batch larger than batch_size: more slots
                     buf(l->partials, (size_t)l->G * grid * l->net.P), buf(l->loss_partials, (size_t)l->G * grid))))
        return g;
    const float *y_in = nullptr;
    if (r.td_fused) {
        y_in = l->y_buf;                                  // not read: the training kernel forms the TD targets itself
    } else if (r.fwd) {
        // TD targets on the tensor cores: y = r + gamma * next_q * (1 - d) for the whole batch, then the training kernel
        // only evaluates the local network (forward on s, backward)
        if ((g.rc = grow(l->td_mem, l->y_cap, B, st, false, buf(l->y_buf, (size_t)l->G * B), buf(l->astar_buf, (size_t)l->G * B))))
            return g;
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.src = src; a.n = B; a.use_next = 1; a.gamma = l->cfg.gamma;
        a.actions = l->astar_buf; a.y_out = l->y_buf;
        if (l->cfg.algo != UAVRL_ALGO_DQN) {             // double DQN: a* = argmax_a q_local(s')
            a.img = l->tc_img_local; a.mode = kTcArgmax;
            if ((g.rc = launch_tc_forward(l, r, a, st))) return g;
            a.mode = kTcTdGather;
        } else {
            a.mode = kTcTdMax;
        }
        a.img = l->tc_img_target;
        if ((g.rc = launch_tc_forward(l, r, a, st))) return g;
        y_in = l->y_buf;
    }
    if ((g.rc = mark(marks, 0, st))) return g;
    if (r.train) {
        // the whole update on the tensor cores: forward + dX chain, then split-K weight gradients (tc_train.cu)
        if ((g.rc = grow(l->rows_mem, l->train_cap, B, st, false,
                         buf(l->act_buf, (size_t)l->G * B * (size_t)(l->tc.act_stride > 0 ? l->tc.act_stride : 4)),
                         buf(l->dz_buf, (size_t)l->G * B * (size_t)l->tc.dz_stride))))
            return g;
        if ((g.rc = launch_tc_train(l, r, src, B, global_batch, y_in, &g.nparts, &g.n_loss_parts, st, marks ? marks[1] : nullptr)))
            return g;
    } else {
        if ((g.rc = launch_fp32_update(l, src, B, global_batch, grid, y_in, st)) || (g.rc = mark(marks, 1, st))) return g;
        g.nparts = g.n_loss_parts = grid;
    }
    g.rc = mark(marks, 2, st);
    return g;
}

// hard_update (DuelingDQN_Trainer.py:199-202): the optimiser step of every update_loop-th epoch also copies local -> target
static int hard_update_due(const uavrl_learner *l) { return (l->cfg.update_loop > 0 && (l->epoch % l->cfg.update_loop) == 0) ? 1 : 0; }

// The optimiser step's arguments for the partials g.  apply: the Adam step follows the reduction; it counts one step and
// copies local -> target when a hard update is due.
static AdamArgs adam_args(uavrl_learner *l, const Grads &g, bool apply)
{
    AdamArgs a;
    memset(&a, 0, sizeof(a));
    a.P = l->net.P; a.nparts = g.nparts; a.n_loss_parts = g.n_loss_parts; a.apply = apply ? 1 : 0; a.world = l->comm.world;
    a.img_floats = l->net.smem_w_floats; a.tc_floats = l->tc.train_img_bytes / 4;
    a.inv_b = g.inv_b;
    if (apply) {
        adam_hyper(a, l->cfg.lr, ++l->adam_t);
        a.hard = hard_update_due(l);
    }
    return a;
}

// reduce_adam_kernel, one grid row per trainer: reduce + Adam, reduce only (a.apply = 0), or Adam on the gradient already in
// l->grad (a.nparts = 0)
static int launch_reduce_adam_step(uavrl_learner *l, const AdamArgs &a, ChainKernel kind, float *loss_out, cudaStream_t st)
{
    UAVRL_CUDA(launch_reduce_adam(l->G, st, l->chain.next(kind).pdl, a, learner_adam_ptrs(l, loss_out)));
    l->chain.launched(kind);
    UAVRL_LAUNCHED();
    return 0;
}

// dp_allreduce_adam_kernel: this rank's partials g summed with every other rank's, then Adam
static int launch_allreduce_adam(uavrl_learner *l, const Grads &g, float *loss_out, cudaStream_t st)
{
    const int P = l->net.P;
    const AdamArgs a = adam_args(l, g, true);
    DpExchange x;                                                               // one rank's slot: gradient vector + loss share
    memset(&x, 0, sizeof(x));
    x.n_seg = 1;
    x.seg[0].partials = l->partials; x.seg[0].nparts = g.nparts; x.seg[0].P = P;
    x.seg[0].q = learner_adam_ptrs(l, loss_out);
    x.extra_parts = l->loss_partials; x.n_extra_parts = g.n_loss_parts; x.extra_stride = 1; x.n_extra = 1;
    x.extra_scale = a.inv_b; x.extra_out = x.seg[0].q.loss_out;
    UAVRL_CUDA(launch_dp_exchange(l->comm, a, x, st, l->chain.next(kChainAdam).pdl));
    l->chain.launched(kChainAdam);
    UAVRL_LAUNCHED();
    return 0;
}

// ReplayTree.batch_update: the |Q - y| of a SumTree-sampled batch become its priorities
static int per_write_back(uavrl_learner *l, const Grads &g, int B, cudaStream_t st)
{
    if (!g.per) return 0;
    if (int rc = l->replay.per_write_back(B, st)) return rc;
    l->chain.launched(kChainNone);
    return 0;
}

int launch_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, bool apply, cudaStream_t st,
                  cudaEvent_t *marks)
{
    const Grads g = launch_grads(l, src, B, global_batch, st, marks);
    if (g.rc) return g.rc;
    if (int rc = launch_reduce_adam_step(l, adam_args(l, g, apply), kChainAdam, loss_out ? loss_out : l->loss_dev, st)) return rc;
    return per_write_back(l, g, B, st);
}

int launch_update_dp(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, cudaStream_t st)
{
    const Grads g = launch_grads(l, src, B, global_batch, st, nullptr);
    if (g.rc) return g.rc;
    if (int rc = launch_allreduce_adam(l, g, loss_out ? loss_out : l->loss_dev, st)) return rc;
    return per_write_back(l, g, B, st);
}

static int repack_images(uavrl_learner *l, cudaStream_t st)
{
    const int threads = 256;
    const dim3 blocks((l->net.P + threads - 1) / threads, l->G);          // y: trainer
    const int wf = l->net.smem_w_floats, tf = l->tc.train_img_bytes / 4;
    pack_image_kernel<<<blocks, threads, 0, st>>>(l->net.P, l->local, l->img_map, l->img_local, wf);
    UAVRL_LAUNCHED();
    pack_image_kernel<<<blocks, threads, 0, st>>>(l->net.P, l->target, l->img_map, l->img_target, wf);
    UAVRL_LAUNCHED();
    if (l->tc_ok) {
        pack_tc_kernel<<<blocks, threads, 0, st>>>(l->net.P, l->local, l->tc_hi_map, l->tc_lo_map, l->tc_hi2_map, l->tc_lo2_map,
                                                   (float *)l->tc_img_local, tf);
        UAVRL_LAUNCHED();
        pack_tc_kernel<<<blocks, threads, 0, st>>>(l->net.P, l->target, l->tc_hi_map, l->tc_lo_map, l->tc_hi2_map, l->tc_lo2_map,
                                                   (float *)l->tc_img_target, tf);
        UAVRL_LAUNCHED();
    }
    return 0;
}

AdamPtrs learner_adam_ptrs(const uavrl_learner *l, float *loss_out)
{
    AdamPtrs q;
    q.partials = l->partials; q.loss_partials = l->loss_partials; q.grad = l->grad; q.local = l->local; q.m = l->m; q.v = l->v;
    q.target = l->target; q.img_local = l->img_local; q.img_target = l->img_target; q.img_map = l->img_map;
    q.tc_local = (float *)l->tc_img_local; q.tc_target = (float *)l->tc_img_target; q.tc_hi = l->tc_hi_map; q.tc_lo = l->tc_lo_map;
    q.tc_hi2 = l->tc_hi2_map; q.tc_lo2 = l->tc_lo2_map; q.loss_out = loss_out;
    return q;
}

// everything uavrl_learner_create_trainers builds; on failure the caller destroys the half-built handle
static int learner_init(uavrl_learner *l, const uavrl_learner_config *cfg, int32_t n_trainers)
{
    l->cfg = *cfg;
    l->G = n_trainers;
    int rc = build_net(*cfg, l->net);
    if (rc) return rc;
    // the fp32 kernels hold the whole network in shared memory: refuse a network that does not fit before allocating anything
    l->dual_weights = upd_smem_bytes(l->net, 1) <= kMaxBlockSmem ? 1 : 0;
    if (upd_smem_bytes(l->net, l->dual_weights) > kMaxBlockSmem || act_smem_bytes(l->net) > kMaxBlockSmem)
        return fail(UAVRL_ERR_INVALID, "network too large for the shared-memory resident kernels");
    const size_t G = (size_t)n_trainers, P = (size_t)l->net.P;
    l->max_ctas = 4 * num_sms();
    l->parts_cap = trainer_parts_cap(n_trainers, cfg->batch_size, l->max_ctas);   // the fp32 update kernel's grid is the widest
    DevMem &m = l->mem, &pm = l->parts_mem;
    if ((rc = m.alloc(l->local, G * P)) || (rc = m.alloc(l->target, G * P)) || (rc = m.alloc(l->m, G * P)) ||
        (rc = m.alloc(l->v, G * P)) || (rc = m.alloc(l->grad, G * P)) ||
        (rc = pm.alloc(l->partials, G * P * (size_t)l->parts_cap)) || (rc = pm.alloc(l->loss_partials, G * (size_t)l->parts_cap)) ||
        (rc = m.alloc(l->loss_dev, G)))
        return rc;
    {
        const size_t wf = (size_t)l->net.smem_w_floats;
        if ((rc = m.alloc(l->img_local, G * wf)) || (rc = m.alloc(l->img_target, G * wf)) || (rc = m.alloc(l->img_map, P))) return rc;
        std::vector<int32_t> map;
        build_image_map(l->net, map);
        UAVRL_CUDA(cudaMemcpy(l->img_map, map.data(), P * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    if ((rc = tc_init(l))) return rc;
    if ((rc = l->replay.alloc(cfg->replay_capacity, cfg->lockstep_envs, n_trainers, cfg->in_dim, false))) return rc;
    if ((rc = raise_dyn_smem(act_kernel_t<false>, act_smem_bytes(l->net))) || (rc = raise_dyn_smem(act_kernel_t<true>, act_smem_bytes(l->net))) || (rc = raise_dyn_smem(update_kernel, upd_smem_bytes(l->net, l->dual_weights))))
        return rc;
    return 0;
}

}  // namespace uavrl

using namespace uavrl;

extern "C" {

int uavrl_learner_create(const uavrl_learner_config *cfg, uavrl_learner **out)
{
    return uavrl_learner_create_trainers(cfg, 1, out);
}

int uavrl_learner_create_trainers(const uavrl_learner_config *cfg, int32_t n_trainers, uavrl_learner **out)
{
    if (!cfg || !out) return fail(UAVRL_ERR_INVALID, "uavrl_learner_create: null argument");
    if (cfg->algo < 0 || cfg->algo > 2) return fail(UAVRL_ERR_INVALID, "unknown algo");
    if (cfg->loss_kind < 0 || cfg->loss_kind > 1) return fail(UAVRL_ERR_INVALID, "loss_kind must be 0 (MSE) or 1 (Huber)");
    if (int rc = check_trainer_group(*cfg, n_trainers, "learner")) return rc;
    uavrl_learner *l = new uavrl_learner();
    if (int rc = learner_init(l, cfg, n_trainers)) { uavrl_learner_destroy(l); return rc; }
    *out = l;
    return 0;
}

int uavrl_learner_destroy(uavrl_learner *l)
{
    if (!l) return 0;
    cudaSetDevice(l->cfg.device);
    cudaDeviceSynchronize();
    delete l;
    return 0;
}

int64_t uavrl_learner_param_count(const uavrl_learner *l) { return l ? l->net.P : 0; }
int32_t uavrl_learner_trainer_count(const uavrl_learner *l) { return l ? l->G : 0; }

static float *which_buf(uavrl_learner *l, int which)
{
    switch (which) {
    case 0: return l->local; case 1: return l->target; case 2: return l->m; case 3: return l->v; case 4: return l->grad;
    default: return nullptr;
    }
}

int uavrl_learner_set_params(uavrl_learner *l, int32_t which, const float *h)
{
    if (!l || !h || !which_buf(l, which)) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(which_buf(l, which), h, (size_t)l->G * l->net.P * 4, cudaMemcpyHostToDevice));
    if (which <= 1) { int rc = repack_images(l, 0); if (rc) return rc; UAVRL_CUDA(cudaDeviceSynchronize()); }
    return 0;
}

int uavrl_learner_get_params(uavrl_learner *l, int32_t which, float *h)
{
    if (!l || !h || !which_buf(l, which)) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(h, which_buf(l, which), (size_t)l->G * l->net.P * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_learner_set_counters(uavrl_learner *l, int64_t epoch, int64_t adam_step)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    l->epoch = epoch; l->adam_t = adam_step;
    return 0;
}

int uavrl_learner_get_counters(uavrl_learner *l, int64_t *epoch, int64_t *adam_step)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (epoch) *epoch = l->epoch;
    if (adam_step) *adam_step = l->adam_t;
    return 0;
}

int uavrl_learner_act(uavrl_learner *l, const float *obs_dev, int32_t n, float eps, int32_t is_train,
                      const float *u_tape_dev, const int32_t *rand_tape_dev, int32_t *actions_dev, float *q_out_dev,
                      void *stream)
{
    if (!l || !obs_dev || !actions_dev || n <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (n % l->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_learner_act: n must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return launch_act(l, obs_dev, n, eps, is_train, u_tape_dev, rand_tape_dev, actions_dev, q_out_dev, (cudaStream_t)stream);
}

int uavrl_replay_push(uavrl_learner *l, int32_t n, const float *obs, const int32_t *act, const float *rew,
                      const float *next_obs, const uint8_t *done, void *stream)
{
    if (!l || n <= 0 || !obs || !act || !rew || !next_obs || !done) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_grouped(l->G, "uavrl_replay_push (grouped learners take the lockstep ring or explicit batches)")) return rc;
    ReplayStore &rs = l->replay;
    if (rs.mode != kReplayPaired) return fail(UAVRL_ERR_STATE, "uavrl_replay_push needs lockstep_envs == 0 (the lockstep ring is fed by uavrl_train_run)");
    if (n > rs.slots) return fail(UAVRL_ERR_INVALID, "push larger than the replay capacity");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    if (int rc = rs.push(n, obs, act, rew, next_obs, done, (cudaStream_t)stream)) return rc;
    if (rs.per_enabled()) l->chain.launched(kChainNone);
    return 0;
}

int64_t uavrl_replay_size(const uavrl_learner *l) { return l ? l->replay.count : 0; }

// kept for ABI compatibility: the lockstep loops always launch get_action and the env step as two kernels
int uavrl_set_fuse_act_env(int32_t on)
{
    return on ? fail(UAVRL_ERR_INVALID, "uavrl_set_fuse_act_env: the fused get_action + env step variant was removed") : 0;
}

int uavrl_replay_gather(uavrl_learner *l, int32_t n, const int64_t *idx, float *s, int32_t *a, float *r, float *s2,
                        uint8_t *d)
{
    if (!l || n <= 0 || !idx) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return l->replay.gather(n, idx, s, a, nullptr, r, s2, d);
}

static int do_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_dev, bool apply, void *stream)
{
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    // one Trainer.update call = TD pass(es) -> training chain -> weight gradients -> optimiser: chain them with PDL
    ChainScope chain(l->chain);
    return launch_update(l, src, B, global_batch, loss_dev, apply, (cudaStream_t)stream);
}

int uavrl_learner_update(uavrl_learner *l, const int32_t *idx_tape_dev, float *loss_dev, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    l->epoch += 1;                                              // DuelingDQN_Trainer.py:152
    if (!l->replay.ready(l->cfg.batch_size)) return 0;          // nothing sampled yet
    BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, idx_tape_dev);
    return do_update(l, src, l->cfg.batch_size, l->cfg.batch_size, loss_dev, true, stream);
}

int uavrl_learner_update_batch(uavrl_learner *l, int32_t B, const float *s, const int32_t *a, const float *r,
                               const float *s2, const float *d, float *loss_dev, void *stream)
{
    if (!l || B <= 0 || !s || !a || !r || !s2 || !d) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (B % l->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_learner_update_batch: B must be a multiple of the trainer count");
    l->epoch += 1;
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kBatchExplicit; src.frames = s; src.s2_rows = s2; src.act = a; src.rew = r; src.done_f32 = d;
    const int Bg = B / l->G;                                    // block g of the rows belongs to trainer g
    return do_update(l, src, Bg, Bg, loss_dev, true, stream);
}

int uavrl_learner_update_batch_per(uavrl_learner *l, int32_t B, const float *s, const int32_t *a, const float *r, const float *s2,
                                   const float *d, const float *is_weights, float *abs_err_out, float *loss_dev, void *stream)
{
    if (!l || B <= 0 || !s || !a || !r || !s2 || !d) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_grouped(l->G, "uavrl_learner_update_batch_per (prioritised replay)")) return rc;
    l->epoch += 1;
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kBatchExplicit; src.frames = s; src.s2_rows = s2; src.act = a; src.rew = r; src.done_f32 = d;
    src.is_w = is_weights; src.abs_err = abs_err_out;
    return do_update(l, src, B, B, loss_dev, true, stream);
}

int uavrl_learner_compute_grads(uavrl_learner *l, const int32_t *idx_tape_dev, int32_t global_batch, float *loss_dev,
                                void *stream)
{
    if (!l || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_grouped(l->G, "uavrl_learner_compute_grads (data-parallel training)")) return rc;
    // refused before the epoch counts: a rank that retries must stay on the other ranks' sample keys and target schedule
    if (!l->replay.ready(l->cfg.batch_size)) return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions");
    l->epoch += 1;
    BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, idx_tape_dev);
    return do_update(l, src, l->cfg.batch_size, global_batch, loss_dev, false, stream);
}

float *uavrl_learner_grad_ptr(uavrl_learner *l) { return l ? l->grad : nullptr; }

int uavrl_learner_apply_grads(uavrl_learner *l, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (int rc = refuse_grouped(l->G, "uavrl_learner_apply_grads (data-parallel training)")) return rc;
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return launch_reduce_adam_step(l, adam_args(l, Grads{}, true), kChainNone, nullptr, (cudaStream_t)stream);
}

int uavrl_learner_hard_update(uavrl_learner *l, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    // every trainer's vectors and images are contiguous ([G][...]): one copy each covers all trainers
    const size_t G = (size_t)l->G;
    const cudaStream_t st = (cudaStream_t)stream;
    launch_copy(G * l->net.P, l->local, l->target, st);
    UAVRL_LAUNCHED();
    launch_copy(G * l->net.smem_w_floats, l->img_local, l->img_target, st);
    UAVRL_LAUNCHED();
    if (l->tc_ok) {
        launch_copy(G * (size_t)(l->tc.train_img_bytes / 4), (const float *)l->tc_img_local, (float *)l->tc_img_target, st);
        UAVRL_LAUNCHED();
    }
    return 0;
}

int uavrl_set_fuse_td(int32_t on) { g_fuse_td.store(on ? 1 : 0); return 0; }
int uavrl_learner_td_fused(const uavrl_learner *l, int32_t batch) { return (l && learner_route(l, batch).td_fused) ? 1 : 0; }

int uavrl_learner_tc_route(const uavrl_learner *l, int32_t n, int32_t *out)
{
    if (!l || !out || n <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    const Route r = learner_route(l, n);
    out[0] = r.fwd; out[1] = r.train; out[2] = r.fwd_rows; out[3] = r.train_rows; out[4] = r.td_fused; out[5] = r.fp32_dual;
    return 0;
}

int uavrl_learner_set_tensor_cores(uavrl_learner *l, int32_t enable)
{
    if (!l) return 0;
    l->use_tc = enable != 0;
    return (l->tc_ok && l->use_tc) ? 1 : 0;
}

int uavrl_learner_set_is_train(uavrl_learner *l, int32_t is_train)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    l->is_train = is_train ? 1 : 0;
    return 0;
}

int uavrl_learner_lockstep_restart(uavrl_learner *l)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (l->replay.mode != kReplayLockstep) return 0;
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return l->replay.restart();
}

// ------------------------------------------------------------------ prioritised replay: the SumTrees of the learner's replay
// store (per.cu).  Their kernels launch outside the dependent-launch chain.
int uavrl_per_enable(uavrl_learner *l, double alpha, double beta0, double beta_inc, double eps, double err_upper)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (l->G > 1) return fail(UAVRL_ERR_INVALID, "prioritised replay is not available on a learner with several trainers");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return l->replay.per_enable(alpha, beta0, beta_inc, eps, err_upper);
}

int uavrl_per_enable_trainers(uavrl_learner *l, double alpha, double beta0, double beta_inc, double eps, double err_upper)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    return l->replay.per_enable(alpha, beta0, beta_inc, eps, err_upper);
}

int uavrl_per_set_priorities(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const double *prio_dev, void *stream)
{
    if (int rc = per_entry_set(l ? &l->replay : nullptr, l ? l->cfg.device : 0, n, slots_dev, prio_dev, nullptr, 0,
                               (cudaStream_t)stream))
        return rc;
    l->chain.launched(kChainNone);
    return 0;
}

int uavrl_per_set_errors(uavrl_learner *l, int32_t n, const int32_t *slots_dev, const float *abs_err_dev, int32_t clip, void *stream)
{
    if (int rc = per_entry_set(l ? &l->replay : nullptr, l ? l->cfg.device : 0, n, slots_dev, nullptr, abs_err_dev, clip, (cudaStream_t)stream))
        return rc;
    l->chain.launched(kChainNone);
    return 0;
}

int uavrl_per_sample(uavrl_learner *l, int32_t B, const double *u_tape_dev, int32_t *slots_out_dev, float *weights_out_dev, void *stream)
{
    if (int rc = per_entry_sample(l ? &l->replay : nullptr, l ? l->cfg.device : 0, l ? l->cfg.seed : 0, B, u_tape_dev, slots_out_dev,
                                  weights_out_dev, (cudaStream_t)stream))
        return rc;
    l->chain.launched(kChainNone);
    return 0;
}

int uavrl_per_get(uavrl_learner *l, double *leaves_host, double *total_out, double *beta_out)
{
    return per_entry_get(l ? &l->replay : nullptr, l ? l->cfg.device : 0, leaves_host, total_out, beta_out);
}

// ------------------------------------------------------------------ fused NVLink all-reduce + Adam
// flag_handle_out / flag_handles: unused (kept for ABI compatibility), may be NULL
int uavrl_learner_comm_init(uavrl_learner *l, int32_t rank, int32_t world, void *grad_handle_out, void *flag_handle_out)
{
    (void)flag_handle_out;
    if (!l) return fail(UAVRL_ERR_INVALID, "bad rank/world/handle pointer");
    if (int rc = refuse_grouped(l->G, "uavrl_learner_comm_init (data-parallel training)")) return rc;
    return comm_init(l->comm, l->cfg.device, rank, world, (size_t)l->net.P + 1, grad_handle_out, false);
}

int uavrl_learner_comm_connect(uavrl_learner *l, const void *grad_handles, const void *flag_handles)
{
    (void)flag_handles;
    if (int rc = refuse_grouped(l ? l->G : 1, "uavrl_learner_comm_connect (data-parallel training)")) return rc;
    if (!l || !grad_handles || !l->comm.recv) return fail(UAVRL_ERR_STATE, "uavrl_learner_comm_connect before comm_init");
    return comm_connect(l->comm, l->cfg.device, grad_handles, false);
}

int uavrl_learner_update_dp(uavrl_learner *l, const int32_t *idx_tape_dev, int32_t global_batch, float *loss_dev, void *stream)
{
    if (!l || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_grouped(l->G, "uavrl_learner_update_dp (data-parallel training)")) return rc;
    if (!l->comm.ready) return fail(UAVRL_ERR_STATE, "uavrl_learner_update_dp before uavrl_learner_comm_connect");
    if (!l->replay.ready(l->cfg.batch_size)) return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    l->epoch += 1;
    BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, idx_tape_dev);
    return launch_update_dp(l, src, l->cfg.batch_size, global_batch, loss_dev, (cudaStream_t)stream);
}

}  // extern "C"
