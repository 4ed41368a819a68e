// learner.cu -- DQN-family learner on device: Q-net forward + eps-greedy, replay ring, sampled
// TD update (forward local/target, MSE, backward), Adam, hard target update.  sm_90a.
//
// Replaces (SURVEY.md section 8a rows a-10..a-13):
//   Trainer.get_action        Trainer/DuelingDQN_Trainer.py:86-97
//   ReplayMemory.add/sample2  BaseClass/replay_buffer.py:41-51
//   Trainer.update            Trainer/DuelingDQN_Trainer.py:150-190, Trainer/DDQN_Trainer.py:72-117,
//                             Trainer/DQN_Trainer.py:85-136
//   networks                  BaseClass/BaseCNN.py:93-102,120-217,329-343
//   torch.optim.Adam step + hard_update (DuelingDQN_Trainer.py:176-184,199-202)
//
// This file is the fp32 CUDA-core path: the whole network (<= 23 k parameters) is staged TRANSPOSED in
// shared memory once per CTA, a CTA owns a tile of 32 samples, lanes walk output units and each
// warp carries 4 samples, so every weight fetch is a conflict-free LDS and every activation fetch
// a broadcast LDS.128.  Gradients leave the CTA as one coalesced partial vector; the optimiser
// kernel reduces the partials in a fixed order (deterministic) and applies Adam.
#include "learner.cuh"
#include "mlp_tile.cuh"
#include "tc_forward.cuh"

#include <math.h>
#include <string.h>

#include <string>
#include <vector>

namespace uavrl {

// ------------------------------------------------------------------ network description (host)
int build_mlp(int in_dim, int n_hidden, const int32_t *hidden, int head_main, int head_extra, NetDev &n)
{
    memset(&n, 0, sizeof(n));
    if (in_dim <= 0 || in_dim > kMaxDim) return fail(UAVRL_ERR_INVALID, "in_dim must be in [1,128]");
    if (n_hidden < 1 || n_hidden > UAVRL_MAX_HIDDEN) return fail(UAVRL_ERR_INVALID, "n_hidden must be in [1,4]");
    if (head_main < 1 || head_main + head_extra > 32) return fail(UAVRL_ERR_INVALID, "head width must be in [1,32]");
    n.in_dim = in_dim; n.n_actions = head_main; n.dueling = 0;
    n.n_layers = n_hidden + 1;
    int in = in_dim, poff = 0, soff = 0;
    for (int l = 0; l < n.n_layers; ++l) {
        LayerDev &L = n.L[l];
        const bool head = (l == n_hidden);
        const int out_real = head ? head_main : hidden[l];
        if (out_real <= 0 || out_real > kMaxDim) return fail(UAVRL_ERR_INVALID, "hidden width must be in [1,128]");
        L.in = in;
        L.out = out_real + (head ? head_extra : 0);
        L.out_main = out_real;
        L.w_off = poff; poff += out_real * in;
        L.b_off = poff; poff += out_real;
        L.w2_off = L.b2_off = -1;
        if (head && head_extra > 0) { L.w2_off = poff; poff += head_extra * in; L.b2_off = poff; poff += head_extra; }
        const int ldw = (L.out % 2 == 0) ? L.out + 1 : L.out;
        L.smem_w = soff; soff += round_up(in, 4) * ldw;
        L.smem_b = soff; soff += round_up(L.out, 4);
        in = out_real;
    }
    n.P = poff;
    n.smem_w_floats = round_up(soff, 4);
    int off = n.smem_w_floats;
    // activation planes: X0 (input), H1..Hn (trunk outputs); ld = round_up(dim,32)
    for (int i = 0; i <= n_hidden; ++i) {
        const int dim = (i == 0) ? in_dim : hidden[i - 1];
        n.act_ld[i] = round_up(dim, 32);
        n.act_off[i] = off; off += kTile * n.act_ld[i];
    }
    n.smem_total_floats = off;   // kernels append their own extra planes after this
    return 0;
}

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
// [S (w + 1), n) of obs = [G][S][in_dim], S = kFedProbes; a tile takes 3 whole probe groups (30 rows) and writes
// fl.loss_out[p][w] = sum over trainer p's rows of sum_a (fl.q_ref - Q_w)^2 / (S A).  The same reduction as the tensor-core
// loss variant (tc_forward.cu).
struct FedLossArgs { const float *q_ref; float *loss_out; int w0, tri; };

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
        params += (size_t)w_set * img_floats; obs += row0 * net.in_dim;
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
                fed_group_loss(sA + threadIdx.x * kFedProbes, row0 + e0 + threadIdx.x * kFedProbes, n, w_set, net.n_actions, fl.loss_out);
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

cudaError_t launch_reduce_adam(dim3 grid, cudaStream_t st, bool pdl, const AdamArgs &a, const AdamPtrs &q)
{
    return launch_kernel(reduce_adam_kernel, grid, dim3(256), 0, st, pdl, a, q.partials, q.loss_partials, q.grad, q.local, q.m, q.v, q.target,
                         q.img_local, q.img_target, q.img_map, q.tc_local, q.tc_target, q.tc_hi, q.tc_lo, q.tc_hi2, q.tc_lo2, q.loss_out);
}

// ---- data-parallel optimiser step: one-shot NVLink all-reduce fused with Adam, in ONE kernel, block by block, with no fence
// and no flag words.  Every rank owns a symmetric receive buffer (slot q belongs to rank q); block b owns parameters
// [64 b, 64 b + 64).  It reduces its slice of this rank's partials and pushes each value into slot `rank` of every rank's
// receive buffer as ONE 8-byte word {epoch : value} (a single-copy-atomic store: the value can never be seen without its
// epoch -- the "LL" idea of NCCL's low-latency protocol).  Then the 64 threads of the block poll -- in local memory -- the
// `world` words of their own parameter until every epoch matches, sum the values in rank order and apply Adam.  A
// __threadfence_system() between data and a flag would cost a system-scope fence per launch even on one GPU; here nothing
// orders two stores, so nothing needs a fence.  recv[2][world][P + 1] alternates by epoch parity: a sender can
// overwrite a slot only two exchanges later, and it cannot finish the exchange in between before the receiver has read.
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
// sum over ranks (fixed order: every rank computes the same bits) of the words {epoch : value} at recv[w * stride]
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

__global__ void __launch_bounds__(256)
dp_allreduce_adam_kernel(AdamArgs a, int nparts, int n_loss_parts, const float *__restrict__ partials,
                         const float *__restrict__ loss_partials, unsigned long long *const *peer_recv,
                         const unsigned long long *recv_local, size_t stride, size_t parity_off, int rank, unsigned epoch,
                         AdamPtrs q, unsigned long long *trace)
{
    // trace (UAVRL_DP_TRACE=1): block 0 accumulates nanoseconds spent in {reduce, push, wait for the peers' words, Adam} and a launch count
    unsigned long long t0 = 0, t1 = 0, t2 = 0, t3 = 0;
    auto now = [] { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };
    __shared__ float red[4][64];
    const int ix = threadIdx.x & 63, cg = threadIdx.x >> 6;
    const int i = blockIdx.x * 64 + ix;
    AdamPre pre;
    if (cg == 0 && i < a.P) pre = adam_prefetch(q, i);   // before the wait: nothing here is the predecessor's output
    pdl_wait();                 // PDL (common.cuh): the gradient partials come from the predecessor
    pdl_trigger();
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t0 = now();
    float g = 0.f;
    if (i < a.P) g = reduce_group(partials, a.P, nparts, i, cg);
    red[cg][ix] = g;
    __syncthreads();
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t1 = now();
    const size_t slot = parity_off + (size_t)rank * stride;
    const unsigned long long tag = (unsigned long long)epoch << 32;
    if (i < a.P) {
        const float gs = (red[0][ix] + red[1][ix]) + (red[2][ix] + red[3][ix]);
        for (int w = cg; w < a.world; w += 4) st_relaxed_sys_u64(peer_recv[w] + slot + i, tag | __float_as_uint(gs));   // 512 contiguous bytes per peer
    }
    if (blockIdx.x == 0 && threadIdx.x >= 224) {                 // last warp of block 0: this rank's loss share
        const int lane = threadIdx.x & 31;
        float s = 0.f;
        for (int c = lane; c < n_loss_parts; c += 32) s += loss_partials[c];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0)
            for (int w = 0; w < a.world; ++w) st_relaxed_sys_u64(peer_recv[w] + slot + a.P, tag | __float_as_uint(s * a.inv_b));
    }
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) t2 = now();
    const unsigned long long *recv = recv_local + parity_off;
    if (cg == 0 && i < a.P) {
        const float gsum = ll_gather_sum(recv + i, stride, a.world, epoch);
        if (trace && blockIdx.x == 0 && threadIdx.x == 0) t3 = now();
        q.grad[i] = gsum;
        adam_update_pre(a, q, i, gsum, pre);
    }
    if (blockIdx.x == 0 && threadIdx.x == 255 && q.loss_out) *q.loss_out = ll_gather_sum(recv + a.P, stride, a.world, epoch);
    if (trace && blockIdx.x == 0) {
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long t4 = now();
            trace[0] += t1 - t0; trace[1] += t2 - t1; trace[2] += t3 - t2; trace[3] += t4 - t3; trace[4] += 1;
        }
    }
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

// generic replay push (paired rows)
__global__ void push_kernel(int n, int in, int64_t head, int64_t cap, const float *__restrict__ obs,
                            const int32_t *__restrict__ act, const float *__restrict__ rew,
                            const float *__restrict__ next_obs, const uint8_t *__restrict__ done,
                            float *__restrict__ frames, int32_t *__restrict__ r_act, float *__restrict__ r_rew,
                            uint8_t *__restrict__ r_done)
{
    const int64_t total = (int64_t)n * in;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i / in, k = i - t * in;
        const int64_t slot = (head + t) % cap;
        frames[(2 * slot) * in + k] = obs[i];
        frames[(2 * slot + 1) * in + k] = next_obs[i];
        if (k == 0) { r_act[slot] = act[t]; r_rew[slot] = rew[t]; r_done[slot] = done[t]; }
    }
}

// ------------------------------------------------------------------ host launchers
static size_t act_smem_bytes(const NetDev &n) { return (size_t)(n.smem_total_floats + 2 * kTile * kMaxDim + kTile * 32) * 4; }
static size_t upd_smem_bytes(const NetDev &n, int dual)
{
    return (size_t)((dual ? n.smem_w_floats : 0) + n.smem_total_floats + kTile * n.act_ld[0] + 2 * kTile * kMaxDim +
                    3 * kTile * 32) * 4;
}
static const size_t kMaxDynSmem = 227 * 1024;

int launch_act(uavrl_learner *l, const float *obs, int n_all, float eps, int is_train, const float *u_tape,
               const int32_t *rand_tape, int32_t *actions, float *q_out, cudaStream_t st)
{
    const int n = n_all / l->G;                          // rows per trainer (grouped learner: G equal blocks)
    if (l->tc_ok && l->use_tc) {                         // tensor-core forward chain (tc_forward.cu)
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.img = l->tc_img_local; a.obs = obs; a.n = n; a.n_tiles = (n + kTcTile - 1) / kTcTile; a.mode = kTcAct;
        a.eps = eps; a.is_train = is_train; a.u_tape = u_tape; a.rand_tape = rand_tape;
        a.key = l->cfg.seed ^ kActSalt; a.call = l->act_calls++; a.actions = actions; a.q_out = q_out;
        return launch_tc_forward(l, a, st);
    }
    const int n_tiles = (n + kTile - 1) / kTile;
    const int grid = n_tiles < 4 * num_sms() ? n_tiles : 4 * num_sms();
    act_kernel_t<false><<<dim3(grid, l->G), kNetThreads, act_smem_bytes(l->net), st>>>(l->net, l->img_local, obs, n, eps, is_train, u_tape,
                                                                                      rand_tape, l->cfg.seed ^ kActSalt, l->act_calls++,
                                                                                      actions, nullptr, q_out, n_tiles, l->net.smem_w_floats,
                                                                                      FedLossArgs{});
    l->pdl_prev = kPdlNone;
    UAVRL_LAUNCHED();
    return 0;
}

int launch_fed_loss(uavrl_learner *l, const float *probes, const float *q_ref, float *loss_out, int w0, int n_weights, bool tri,
                    cudaStream_t st)
{
    const int n = l->G * kFedProbes;                     // every probe row; a weight set evaluates at most n - S of them
    const int max_rows = n - kFedProbes;
    if (max_rows <= 0 || n_weights <= 0) return 0;
    if (l->tc_ok && l->use_tc) {
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.img = l->tc_img_local; a.obs = probes; a.n = n; a.mode = kTcAct;
        a.q_ref = q_ref; a.loss_out = loss_out; a.loss_w0 = w0; a.loss_tri = tri ? 1 : 0;
        return launch_tc_loss(l, a, n_weights, max_rows, st);
    }
    constexpr int step = (kTile / kFedProbes) * kFedProbes;
    const int n_tiles = (max_rows + step - 1) / step;
    const int grid = n_tiles < 4 * num_sms() ? n_tiles : 4 * num_sms();
    act_kernel_t<true><<<dim3(grid, n_weights), kNetThreads, act_smem_bytes(l->net), st>>>(l->net, l->img_local, probes, n, 0.f, 0, nullptr,
                                                                                          nullptr, 0, 0, nullptr, nullptr, nullptr, n_tiles,
                                                                                          l->net.smem_w_floats, FedLossArgs{ q_ref, loss_out, w0, tri ? 1 : 0 });
    l->pdl_prev = kPdlNone;
    UAVRL_LAUNCHED();
    return 0;
}

static int launch_update_impl(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, bool apply,
                              cudaStream_t st, cudaEvent_t *mid, bool partials_only = false);

// hard_update (DuelingDQN_Trainer.py:199-202): the optimiser step of every update_loop-th epoch also copies local -> target
static int hard_update_due(const uavrl_learner *l) { return (l->cfg.update_loop > 0 && (l->epoch % l->cfg.update_loop) == 0) ? 1 : 0; }

int launch_update(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, bool apply,
                  cudaStream_t st)
{
    return launch_update_impl(l, src, B, global_batch, loss_out, apply, st, nullptr);
}

// profiling form: mid[0] after the TD-target pass, mid[1] after the forward/backward kernel, mid[2] after the
// weight-gradient kernel (== mid[1] on the CUDA-core path); the optimiser kernel follows
int launch_update_split(uavrl_learner *l, const BatchSrc &src, int B, cudaStream_t st, cudaEvent_t *mid)
{
    return launch_update_impl(l, src, B, B, l->loss_dev, true, st, mid);
}

static int launch_update_impl(uavrl_learner *l, const BatchSrc &src_in, int B, int global_batch, float *loss_out, bool apply,
                              cudaStream_t st, cudaEvent_t *mid, bool partials_only)
{
    BatchSrc src = src_in;
    const bool per_batch = l->per.enabled && src.mode != kBatchExplicit && !src.idx_tape;
    if (per_batch) {
        // ReplayTree.sample2 -> slots + importance weights; |Q - y| comes back for batch_update (end of this function).
        // Grouped learner: [G][B] trainer-local slots, weights and errors; trainer_src hands trainer g its row of each
        int rc = per_sample(l, B, nullptr, nullptr, nullptr, st);
        if (rc) return rc;
        src.idx_tape = l->per.idx; src.idx_is_slot = 1; src.is_w = l->per.w; src.abs_err = l->per.abs_err;
    }
    const int n_tiles = (B + kTile - 1) / kTile;
    const int grid = n_tiles < l->max_ctas ? n_tiles : l->max_ctas;
    if (grid > l->parts_cap) {                           // grouped learner, batch larger than batch_size: more partial slots
        UAVRL_CUDA(cudaStreamSynchronize(st));
        cudaFree(l->partials); cudaFree(l->loss_partials);
        l->partials = nullptr; l->loss_partials = nullptr;
        int rc;
        if ((rc = dev_alloc(&l->partials, (size_t)l->G * grid * l->net.P)) || (rc = dev_alloc(&l->loss_partials, (size_t)l->G * grid)))
            return rc;
        l->parts_cap = grid;
    }
    const float *y_in = nullptr;
    const bool fuse_td = l->tc_ok && l->use_tc && tc_train_can_fuse_td(l, B);
    if (l->tc_ok && l->use_tc && fuse_td) {
        y_in = l->y_buf;                                  // not read: the training kernel forms the TD targets itself
    } else if (l->tc_ok && l->use_tc) {
        // TD targets on the tensor cores: y = r + gamma * next_q * (1 - d) for the whole batch, then the
        // update kernel only evaluates the local network (forward on s, backward)
        if (B > l->y_cap) {
            UAVRL_CUDA(cudaStreamSynchronize(st));
            cudaFree(l->y_buf); cudaFree(l->astar_buf);
            UAVRL_CUDA(cudaMalloc((void **)&l->y_buf, (size_t)l->G * B * 4));
            UAVRL_CUDA(cudaMalloc((void **)&l->astar_buf, (size_t)l->G * B * 4));
            l->y_cap = B;
        }
        TcArgs a;
        memset(&a, 0, sizeof(a));
        a.src = src; a.n = B; a.n_tiles = (B + kTcTile - 1) / kTcTile; a.use_next = 1; a.gamma = l->cfg.gamma;
        a.actions = l->astar_buf; a.y_out = l->y_buf;
        int rc;
        if (l->cfg.algo != UAVRL_ALGO_DQN) {             // double DQN: a* = argmax_a q_local(s')
            a.img = l->tc_img_local; a.mode = kTcArgmax;
            if ((rc = launch_tc_forward(l, a, st))) return rc;
            a.mode = kTcTdGather;
        } else {
            a.mode = kTcTdMax;
        }
        a.img = l->tc_img_target;
        if ((rc = launch_tc_forward(l, a, st))) return rc;
        y_in = l->y_buf;
    }
    if (mid) UAVRL_CUDA(cudaEventRecord(mid[0], st));
    int nparts = grid, n_loss_parts = grid;
    AdamArgs a;
    memset(&a, 0, sizeof(a));
    a.P = l->net.P; a.apply = apply ? 1 : 0; a.world = l->world;
    a.img_floats = l->net.smem_w_floats; a.tc_floats = l->tc.train_img_bytes / 4;
    a.inv_b = 1.0f / (float)global_batch;
    if (apply && !partials_only) {
        adam_hyper(a, l->cfg.lr, ++l->adam_t);
        a.hard = hard_update_due(l);
    }
    if (y_in && l->tc_train_ok) {
        // the whole update on the tensor cores: forward + dX chain, then split-K weight gradients (tc_train.cu)
        if (B > l->train_cap) {
            UAVRL_CUDA(cudaStreamSynchronize(st));
            cudaFree(l->act_buf); cudaFree(l->dz_buf);
            UAVRL_CUDA(cudaMalloc((void **)&l->act_buf, (size_t)l->G * B * (size_t)(l->tc.act_stride > 0 ? l->tc.act_stride : 4) * 4));
            UAVRL_CUDA(cudaMalloc((void **)&l->dz_buf, (size_t)l->G * B * (size_t)l->tc.dz_stride * 4));
            l->train_cap = B;
        }
        int rc = launch_tc_train(l, src, B, global_batch, y_in, &nparts, &n_loss_parts, st, mid ? mid[1] : nullptr, fuse_td);
        if (rc) return rc;
    } else {
    UpdateArgs ua;
    ua.img_local = l->img_local; ua.img_target = l->img_target; ua.partials = l->partials; ua.loss_partials = l->loss_partials;
    ua.B = B; ua.n_tiles = n_tiles; ua.algo = l->cfg.algo; ua.gamma = l->cfg.gamma; ua.dual = l->dual_weights;
    ua.loss_kind = l->cfg.loss_kind; ua.img_floats = l->net.smem_w_floats;
    ua.inv_global_b = 1.0f / (float)global_batch;
    ua.y_in = y_in;
    update_kernel<<<dim3(grid, l->G), kNetThreads, upd_smem_bytes(l->net, l->dual_weights), st>>>(l->net, src, ua);
    l->pdl_prev = kPdlNone;
    UAVRL_LAUNCHED();
    if (mid) UAVRL_CUDA(cudaEventRecord(mid[1], st));
    }
    if (mid) UAVRL_CUDA(cudaEventRecord(mid[2], st));
    l->last_nparts = nparts;
    l->last_n_loss_parts = n_loss_parts;
    l->last_global_batch = global_batch;
    if (partials_only) {                                        // the data-parallel pair follows (launch_update_dp)
        if (per_batch) return per_set(l, B, l->per.idx, nullptr, l->per.abs_err, 1, st);
        return 0;
    }
    a.nparts = nparts; a.n_loss_parts = n_loss_parts;
    const bool chain = l->pdl_chain && g_pdl.load();
    UAVRL_CUDA(launch_reduce_adam(dim3((a.P + 63) / 64, l->G), st, chain && l->pdl_prev == kPdlDw && !mid, a,
                                  learner_adam_ptrs(l, loss_out ? loss_out : l->loss_dev)));
    l->pdl_prev = chain ? kPdlAdam : kPdlNone;
    UAVRL_LAUNCHED();
    if (per_batch) return per_set(l, B, l->per.idx, nullptr, l->per.abs_err, 1, st);      // ReplayTree.batch_update
    return 0;
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

// local gradient partials (same kernels as the single-GPU update, no optimiser step), then the exchange fused with Adam
// (dp_allreduce_adam_kernel)
int launch_update_dp(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, float *loss_out, cudaStream_t st)
{
    int rc = launch_update_impl(l, src, B, global_batch, nullptr, false, st, nullptr, true);
    if (rc) return rc;
    l->comm_epoch += 1;
    const int P = l->net.P;
    const size_t stride = (size_t)P + 1;                                        // one rank's slot: gradient vector + loss share
    const size_t parity_off = (size_t)(l->comm_epoch & 1u) * (size_t)l->world * stride;
    const bool chain = l->pdl_chain && g_pdl.load();
    AdamArgs a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.apply = 1; a.world = l->world;
    adam_hyper(a, l->cfg.lr, ++l->adam_t);
    a.hard = hard_update_due(l);
    a.inv_b = 1.0f / (float)global_batch;
    static const bool dp_trace = getenv("UAVRL_DP_TRACE") != nullptr;
    if (dp_trace && !l->dp_trace) { UAVRL_CUDA(cudaMalloc((void **)&l->dp_trace, 5 * 8)); UAVRL_CUDA(cudaMemsetAsync(l->dp_trace, 0, 40, st)); }
    const int nblk = (P + 63) / 64;
    UAVRL_CUDA(launch_kernel(dp_allreduce_adam_kernel, dim3(nblk), dim3(256), 0, st, chain && l->pdl_prev == kPdlDw, a, l->last_nparts,
                             l->last_n_loss_parts, (const float *)l->partials, (const float *)l->loss_partials,
                             (unsigned long long *const *)l->peer_grad_dev, (const unsigned long long *)l->comm_grad, stride, parity_off,
                             l->rank, l->comm_epoch, learner_adam_ptrs(l, loss_out ? loss_out : l->loss_dev), l->dp_trace));
    UAVRL_LAUNCHED();
    l->pdl_prev = chain ? kPdlAdam : kPdlNone;
    return 0;
}

void lockstep_commit(uavrl_learner *l, cudaStream_t st)
{
    if (l->per.enabled) {
        // the frame just completed becomes sampleable with the priority of an error-less push; the frame that now
        // receives the next observations (the ring's oldest) stops being a transition.  Trainer-local slots: every trainer's
        // tree gets the same Ng + Ng slots of its own env block
        const int64_t Ng = l->replay.N / l->G;
        per_fill_range(l, l->replay.head * Ng, 2 * Ng, per_new_priority(l->per), st, Ng, 0.0);
        l->pdl_prev = kPdlNone;
    }
    l->replay.commit();
}

void adam_hyper(AdamArgs &a, float lr, int64_t t)
{
    const double b1 = 0.9, b2 = 0.999;
    const double bc1 = 1.0 - pow(b1, (double)t), bc2 = 1.0 - pow(b2, (double)t);
    a.step_size = (float)((double)lr / bc1);
    a.beta1_c = (float)(1.0 - b1); a.beta2 = (float)b2; a.beta2_c = (float)(1.0 - b2);
    a.eps = 1e-8f; a.bc2_sqrt = (float)sqrt(bc2);
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
    if (n_trainers < 1 || n_trainers > 65535)        // every grouped kernel runs one grid row per trainer: gridDim.y <= 65535
        return fail(UAVRL_ERR_INVALID, "n_trainers must be in [1, 65535]");
    if (n_trainers > 1 && (cfg->lockstep_envs < 0 || cfg->lockstep_envs % n_trainers != 0))
        return fail(UAVRL_ERR_INVALID, "lockstep_envs must be a multiple of n_trainers (every trainer owns lockstep_envs / n_trainers envs)");
    if (n_trainers > 1 && cfg->replay_capacity / n_trainers <= 0)
        return fail(UAVRL_ERR_INVALID, "replay_capacity / n_trainers must be > 0");
    if (cfg->batch_size <= 0 || cfg->replay_capacity <= 0) return fail(UAVRL_ERR_INVALID, "batch_size and replay_capacity must be > 0");
    if (cfg->algo < 0 || cfg->algo > 2) return fail(UAVRL_ERR_INVALID, "unknown algo");
    if (cfg->loss_kind < 0 || cfg->loss_kind > 1) return fail(UAVRL_ERR_INVALID, "loss_kind must be 0 (MSE) or 1 (Huber)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(UAVRL_ERR_CUDA, "no CUDA device: the learner has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg->device));
    uavrl_learner *l = new uavrl_learner();
    l->cfg = *cfg;
    l->G = n_trainers;
    int rc = build_net(*cfg, l->net);
    if (rc) { delete l; return rc; }
    // the fp32 kernels hold the whole network in shared memory: refuse a network that does not fit before allocating anything
    l->dual_weights = upd_smem_bytes(l->net, 1) <= kMaxDynSmem ? 1 : 0;
    if (upd_smem_bytes(l->net, l->dual_weights) > kMaxDynSmem || act_smem_bytes(l->net) > kMaxDynSmem) {
        delete l;
        return fail(UAVRL_ERR_INVALID, "network too large for the shared-memory resident kernels");
    }
    const size_t G = (size_t)n_trainers, P = (size_t)l->net.P;
    l->max_ctas = 4 * num_sms();
    // gradient / loss partial slots per trainer: one learner keeps max_ctas (any batch); a grouped learner sizes them from the
    // per-trainer batch (the fp32 update kernel's grid, the largest of the update routes) and grows them for larger batches
    {
        const int tiles = (cfg->batch_size + kTile - 1) / kTile;
        l->parts_cap = (G == 1 || tiles > l->max_ctas) ? l->max_ctas : tiles;
    }
    if ((rc = dev_alloc(&l->local, G * P)) || (rc = dev_alloc(&l->target, G * P)) || (rc = dev_alloc(&l->m, G * P)) ||
        (rc = dev_alloc(&l->v, G * P)) || (rc = dev_alloc(&l->grad, G * P)) ||
        (rc = dev_alloc(&l->partials, G * P * (size_t)l->parts_cap)) || (rc = dev_alloc(&l->loss_partials, G * (size_t)l->parts_cap)) ||
        (rc = dev_alloc(&l->loss_dev, G)))
        return rc;
    {
        const size_t wf = (size_t)l->net.smem_w_floats;
        if ((rc = dev_alloc(&l->img_local, G * wf)) || (rc = dev_alloc(&l->img_target, G * wf)) || (rc = dev_alloc(&l->img_map, P))) return rc;
        std::vector<int32_t> map;
        build_image_map(l->net, map);
        UAVRL_CUDA(cudaMemcpy(l->img_map, map.data(), P * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    if ((rc = tc_init(l))) return rc;
    if ((rc = l->replay.alloc(cfg->replay_capacity, cfg->lockstep_envs, n_trainers, cfg->in_dim, false))) return rc;
    if ((rc = raise_dyn_smem(act_kernel_t<false>, act_smem_bytes(l->net))) || (rc = raise_dyn_smem(act_kernel_t<true>, act_smem_bytes(l->net))) || (rc = raise_dyn_smem(update_kernel, upd_smem_bytes(l->net, l->dual_weights))))
        return rc;
    *out = l;
    return 0;
}

int uavrl_learner_destroy(uavrl_learner *l)
{
    if (!l) return 0;
    cudaSetDevice(l->cfg.device);
    cudaDeviceSynchronize();
    if (l->dp_trace) {
        unsigned long long h[5] = { 0, 0, 0, 0, 0 };
        cudaMemcpy(h, l->dp_trace, sizeof(h), cudaMemcpyDeviceToHost);
        if (h[4]) fprintf(stderr, "[dp_trace] rank %d/%d: %llu launches, block 0 mean ns: reduce %.0f  push %.0f  wait for peers' words %.0f  adam %.0f\n",
                          l->rank, l->world, h[4], (double)h[0] / h[4], (double)h[1] / h[4], (double)h[2] / h[4], (double)h[3] / h[4]);
        cudaFree(l->dp_trace);
    }
    for (int q = 0; q < l->world && l->comm_ready; ++q) {
        if (q == l->rank) continue;
        if (l->peer_grad_host[q]) cudaIpcCloseMemHandle(l->peer_grad_host[q]);
    }
    l->replay.release();
    void *ptrs[] = { l->local, l->target, l->m, l->v, l->grad, l->partials, l->loss_partials, l->loss_dev, l->comm_grad, l->peer_grad_dev, l->img_local, l->img_target,
                     l->img_map, l->tc_img_local, l->tc_img_target, l->tc_hi_map, l->tc_lo_map, l->y_buf, l->astar_buf, l->tc_hi2_map,
                     l->tc_lo2_map, l->act_buf, l->dz_buf };
    for (void *p : ptrs) cudaFree(p);
    per_free(l);
    delete l;
    return 0;
}

int64_t uavrl_learner_param_count(const uavrl_learner *l) { return l ? l->net.P : 0; }
int32_t uavrl_learner_trainer_count(const uavrl_learner *l) { return l ? l->G : 0; }

// entry points a grouped learner does not offer: refused before anything is enqueued or allocated
static int refuse_grouped(const uavrl_learner *l, const char *what)
{
    if (l && l->G > 1)
        return fail(UAVRL_ERR_INVALID, std::string(what) + " is not available on a learner with " + std::to_string(l->G) + " trainers");
    return 0;
}

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
    if (int rc = refuse_grouped(l, "uavrl_replay_push (grouped learners take the lockstep ring or explicit batches)")) return rc;
    ReplayStore &rs = l->replay;
    if (rs.mode != kReplayPaired) return fail(UAVRL_ERR_STATE, "uavrl_replay_push needs lockstep_envs == 0 (the lockstep ring is fed by uavrl_train_run)");
    if (n > rs.slots) return fail(UAVRL_ERR_INVALID, "push larger than the replay capacity");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    const int64_t total = (int64_t)n * l->net.in_dim;
    const int threads = 256;
    int blocks = (int)((total + threads - 1) / threads);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    push_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(n, l->net.in_dim, rs.head, rs.slots, obs, act, rew, next_obs,
                                                             done, rs.frames, rs.act, rs.rew, rs.done);
    UAVRL_LAUNCHED();
    if (l->per.enabled) {                                       // ReplayTree.push with error 0; uavrl_per_set_errors refines it
        int rc = per_fill_range(l, rs.head, n, per_new_priority(l->per), (cudaStream_t)stream);
        if (rc) return rc;
    }
    rs.head = (rs.head + n) % rs.slots;
    rs.count = (rs.count + n > rs.slots) ? rs.slots : rs.count + n;
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
    // (the first kernel is launched plainly: whatever precedes it on the stream is not ours)
    const bool outer = l->pdl_chain;
    if (!outer) { l->pdl_chain = true; l->pdl_prev = kPdlNone; }
    const int rc = launch_update(l, src, B, global_batch, loss_dev, apply, (cudaStream_t)stream);
    if (!outer) { l->pdl_chain = false; l->pdl_prev = kPdlNone; }
    return rc;
}

int uavrl_learner_update(uavrl_learner *l, const int32_t *idx_tape_dev, float *loss_dev, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    l->epoch += 1;                                              // DuelingDQN_Trainer.py:152
    if (l->replay.count / l->G <= l->cfg.batch_size) return 0;  // PathPlan_City.py:383: nothing sampled yet (per trainer)
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
    if (int rc = refuse_grouped(l, "uavrl_learner_update_batch_per (prioritised replay)")) return rc;
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
    if (int rc = refuse_grouped(l, "uavrl_learner_compute_grads (data-parallel training)")) return rc;
    // refused before the epoch counts: a rank that retries must stay on the other ranks' sample keys and target schedule
    if (l->replay.count <= l->cfg.batch_size) return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions");
    l->epoch += 1;
    BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, idx_tape_dev);
    return do_update(l, src, l->cfg.batch_size, global_batch, loss_dev, false, stream);
}

float *uavrl_learner_grad_ptr(uavrl_learner *l) { return l ? l->grad : nullptr; }

int uavrl_learner_apply_grads(uavrl_learner *l, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (int rc = refuse_grouped(l, "uavrl_learner_apply_grads (data-parallel training)")) return rc;
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    AdamArgs a;
    memset(&a, 0, sizeof(a));
    a.P = l->net.P; a.nparts = 0; a.apply = 1;
    adam_hyper(a, l->cfg.lr, ++l->adam_t);
    a.hard = hard_update_due(l);
    UAVRL_CUDA(launch_reduce_adam(dim3((a.P + 63) / 64), (cudaStream_t)stream, false, a, learner_adam_ptrs(l, nullptr)));
    UAVRL_LAUNCHED();
    return 0;
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
    l->replay.restart();
    if (l->per.enabled) {
        UAVRL_CUDA(cudaSetDevice(l->cfg.device));
        UAVRL_CUDA(cudaDeviceSynchronize());
        const size_t G = (size_t)l->per.G;                     // every trainer's tree
        UAVRL_CUDA(cudaMemset(l->per.leaf, 0, G * l->per.cap * 8));
        UAVRL_CUDA(cudaMemset(l->per.l1, 0, G * l->per.n1 * 8));
        UAVRL_CUDA(cudaMemset(l->per.l2, 0, G * l->per.n2 * 8));
    }
    return 0;
}

// ------------------------------------------------------------------ fused NVLink all-reduce + Adam
// flag_handle_out / flag_handles: unused (kept for ABI compatibility), may be NULL
int uavrl_learner_comm_init(uavrl_learner *l, int32_t rank, int32_t world, void *grad_handle_out, void *flag_handle_out)
{
    (void)flag_handle_out;
    if (!l || world < 1 || world > 64 || rank < 0 || rank >= world || !grad_handle_out)
        return fail(UAVRL_ERR_INVALID, "bad rank/world/handle pointer");
    if (int rc = refuse_grouped(l, "uavrl_learner_comm_init (data-parallel training)")) return rc;
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    l->rank = rank; l->world = world;
    if (l->comm_grad && l->comm_world != world) {                // re-initialised with another world size
        UAVRL_CUDA(cudaDeviceSynchronize());
        cudaFree(l->comm_grad);
        l->comm_grad = nullptr;
    }
    l->comm_world = world;
    if (!l->comm_grad) {
        // recv[2][world][P+1] words of 8 bytes {epoch : value} (epoch 0 = never written)
        const size_t n = 2 * (size_t)world * ((size_t)l->net.P + 1);
        UAVRL_CUDA(cudaMalloc((void **)&l->comm_grad, n * sizeof(unsigned long long)));
        UAVRL_CUDA(cudaMemset(l->comm_grad, 0, n * sizeof(unsigned long long)));
    }
    cudaIpcMemHandle_t hg;
    UAVRL_CUDA(cudaIpcGetMemHandle(&hg, l->comm_grad));
    memcpy(grad_handle_out, &hg, sizeof(hg));
    return 0;
}

int uavrl_learner_comm_connect(uavrl_learner *l, const void *grad_handles, const void *flag_handles)
{
    (void)flag_handles;
    if (int rc = refuse_grouped(l, "uavrl_learner_comm_connect (data-parallel training)")) return rc;
    if (!l || !grad_handles || !l->comm_grad) return fail(UAVRL_ERR_STATE, "uavrl_learner_comm_connect before comm_init");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    for (int q = 0; q < l->world; ++q) {
        if (q == l->rank) { l->peer_grad_host[q] = l->comm_grad; continue; }
        cudaIpcMemHandle_t hg;
        memcpy(&hg, (const char *)grad_handles + (size_t)q * sizeof(hg), sizeof(hg));
        UAVRL_CUDA(cudaIpcOpenMemHandle(&l->peer_grad_host[q], hg, cudaIpcMemLazyEnablePeerAccess));
    }
    cudaFree(l->peer_grad_dev);
    UAVRL_CUDA(cudaMalloc((void **)&l->peer_grad_dev, sizeof(void *) * l->world));
    UAVRL_CUDA(cudaMemcpy(l->peer_grad_dev, l->peer_grad_host, sizeof(void *) * l->world, cudaMemcpyHostToDevice));
    l->comm_ready = true;
    return 0;
}

int uavrl_learner_update_dp(uavrl_learner *l, const int32_t *idx_tape_dev, int32_t global_batch, float *loss_dev, void *stream)
{
    if (!l || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_grouped(l, "uavrl_learner_update_dp (data-parallel training)")) return rc;
    if (!l->comm_ready) return fail(UAVRL_ERR_STATE, "uavrl_learner_update_dp before uavrl_learner_comm_connect");
    if (l->replay.count <= l->cfg.batch_size) return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    l->epoch += 1;
    BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, idx_tape_dev);
    return launch_update_dp(l, src, l->cfg.batch_size, global_batch, loss_dev, (cudaStream_t)stream);
}

}  // extern "C"
