// tc_forward.cu -- the Q-network forward chain on the Hopper tensor cores (wgmma), sm_90a.
//
// Used for Trainer.get_action (Trainer/DuelingDQN_Trainer.py:86-97) and for the TD-target part of
// Trainer.update (target-network forward, :164-171; DQN_Trainer.py:109; DDQN_Trainer.py:94-95).
//
// One CTA = one tile of up to 128 samples (two warpgroups of m64).  The whole network lives in SMEM as B operands in the
// canonical K-major layout, pre-split into TF32 hi/lo images that the optimiser kernel keeps current
// (one TMA bulk copy stages it).  Per layer:   D[128 x N] (fp32) = A[128 x K] * W[N x K]^T
// issued by each warpgroup as 3 x K/8 `wgmma.mma_async ... tf32` per 64-column chunk (hi*hi + hi*lo + lo*hi: the 3xTF32
// split, fp32 grade, so results stay inside the parity tolerance of the fp32 path).
// The accumulator is staged in a shared-memory tile; the epilogue adds the bias, applies ReLU, re-splits and writes
// the next layer's A operand straight back into SMEM -- activations never touch HBM.  The head's epilogue
// forms Q (dueling combine), then eps-greedy / argmax / max / gather depending on the mode.  The chain itself (gather,
// epilogues, layer loop, head, staging) is tc_chain.cuh, shared with the training kernel's fused TD pass (tc_train.cu).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "tc_chain.cuh"

namespace uavrl {

static inline int rup(int x, int m) { return (x + m - 1) / m * m; }

size_t tc_smem_bytes(const TcNet &tc) { return (size_t)2 * tc.a_bytes + (size_t)tc.img_bytes + (size_t)tc.max_rows * tc.acc_ld * 4; }

int tc_build(const uavrl_learner_config &c, const NetDev &net, TcNet &tc, std::vector<int32_t> &hi_map, std::vector<int32_t> &lo_map,
             std::vector<int32_t> &hi2_map, std::vector<int32_t> &lo2_map)
{
    memset(&tc, 0, sizeof(tc));
    tc.n_layers = net.n_layers; tc.in_dim = net.in_dim; tc.n_actions = net.n_actions; tc.dueling = net.dueling;
    if (net.in_dim % 4 != 0) return -1;
    int off = 0, maxK = 0, k_pad = rup(net.in_dim, 8);
    for (int l = 0; l < net.n_layers; ++l) {
        const LayerDev &L = net.L[l];
        TcLayer &T = tc.L[l];
        const bool head = (l == net.n_layers - 1);
        T.K_real = L.in; T.K_pad = k_pad; T.N_real = L.out;
        T.N_pad = head ? 32 : rup(L.out, 16);
        if (T.N_pad > 128 || T.K_pad > 128 || (head && L.out > 32)) return -1;
        const int bytes = T.N_pad * T.K_pad * 4;
        T.hi_off = off; off += bytes;
        T.lo_off = off; off += bytes;
        if (T.K_pad > maxK) maxK = T.K_pad;
        T.w_off = L.w_off; T.b_off = L.b_off; T.w2_off = L.w2_off; T.b2_off = L.b2_off;
        T.out_main = L.out_main;
        k_pad = T.N_pad;
    }
    tc.bias_base = off;
    int boff = 0;
    for (int l = 0; l < net.n_layers; ++l) { tc.L[l].bias_off = boff; boff += tc.L[l].N_pad; }
    tc.img_bytes = rup(off + boff * 4, 16);
    // transposed blocks for the dX chain (layers >= 1): B' = W^T, rows = input units (K_pad), reduction = outputs (N_pad)
    int toff = tc.img_bytes;
    for (int l = 0; l < net.n_layers; ++l) {
        TcLayer &T = tc.L[l];
        T.t_hi_off = T.t_lo_off = -1;
        if (l == 0) continue;
        const int bytes = T.K_pad * T.N_pad * 4;
        T.t_hi_off = toff; toff += bytes;
        T.t_lo_off = toff; toff += bytes;
    }
    tc.train_img_bytes = rup(toff, 16);
    tc.max_k = maxK;
    {   // accumulator tile: the epilogues read 32-column chunks; + 4 floats so that 16-byte reads of 8 rows hit 32 banks
        int maxN = 32;
        for (int l = 0; l < net.n_layers; ++l) if (tc.L[l].N_pad > maxN) maxN = tc.L[l].N_pad;
        tc.acc_ld = rup(maxN, 32) + 4;
    }
    tc.max_rows = kTcTile;
    tc.a_bytes = (int)mma_tile_bytes(tc.max_rows, maxK);
    if (tc_smem_bytes(tc) + 4096 > kMaxBlockSmem) {              // 128 rows of operands + accumulator, weights, static smem
        tc.max_rows = 64;
        tc.a_bytes = (int)mma_tile_bytes(tc.max_rows, maxK);
    }
    // per-sample scratch: act = inputs of layers 1.. (K_pad each), dz = output derivatives of every layer (N_pad each)
    int ao = 0, dzo = 0;
    for (int l = 0; l < net.n_layers; ++l) {
        tc.L[l].act_off = (l == 0) ? -1 : ao;
        if (l > 0) ao += tc.L[l].K_pad;
        tc.L[l].dz_off = dzo; dzo += tc.L[l].N_pad;
    }
    tc.act_stride = ao; tc.dz_stride = dzo;
    // parameter -> image maps (float indices)
    hi_map.assign((size_t)net.P, -1); lo_map.assign((size_t)net.P, -1);
    hi2_map.assign((size_t)net.P, -1); lo2_map.assign((size_t)net.P, -1);
    auto elem = [](int k_pad_cols, int base, int n, int k) {     // float index of element (row n, col k), K-major canonical
        const int sbo = (k_pad_cols / 4) * 128;
        return (base + (n >> 3) * sbo + (k >> 2) * 128 + (n & 7) * 16 + (k & 3) * 4) / 4;
    };
    for (int l = 0; l < net.n_layers; ++l) {
        const LayerDev &L = net.L[l];
        const TcLayer &T = tc.L[l];
        const int out_main = T.out_main;
        for (int o = 0; o < L.out; ++o) {
            const bool vrow = (o >= out_main);                   // dueling value row
            for (int k = 0; k < L.in; ++k) {
                const size_t pi = vrow ? (size_t)L.w2_off + (size_t)(o - out_main) * L.in + k : (size_t)L.w_off + (size_t)o * L.in + k;
                hi_map[pi] = elem(T.K_pad, T.hi_off, o, k);
                lo_map[pi] = elem(T.K_pad, T.lo_off, o, k);
                if (l > 0) {                                      // W^T: row k, column o
                    hi2_map[pi] = elem(T.N_pad, T.t_hi_off, k, o);
                    lo2_map[pi] = elem(T.N_pad, T.t_lo_off, k, o);
                }
            }
            hi_map[vrow ? (size_t)L.b2_off + (o - out_main) : (size_t)L.b_off + o] = tc.bias_base / 4 + T.bias_off + o;
        }
    }
    (void)c;
    return 0;
}


// ACT (a.mode == kTcAct) and DUELING are compile-time: the kernel a pass runs carries no code of the other modes.
// FIXED: every layer product is one unbroken compile-time wgmma chain (wgmma.cuh mma_fixed; tc_fixed_chains).
// LOSS (with ACT, federation): grid row y evaluates weight set loss_w0 + y on a probe-row range (TcArgs::loss_*); a tile
// takes whole groups of kFedProbes rows, and its head epilogue reduces each group to one loss entry.
// The kernels below are thin entry points over this body: tc_forward_kernel_t (LOSS = false) and tc_loss_kernel_t.
template <bool ACT, bool DUELING, bool FIXED, bool LOSS>
__device__ __forceinline__ void tc_forward_body(const TcNet &tc, const TcArgs &a)
{
    stage_trace(a.trace, 0);
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *Ahi = smem, *Alo = smem + tc.a_bytes, *W = smem + 2 * tc.a_bytes;
    float *acc = reinterpret_cast<float *>(W + tc.img_bytes);        // accumulator tile [tc.max_rows][tc.acc_ld]
    __shared__ uint64_t wbar, wbar2;                         // weights of layer 0 | every other layer + the biases
    __shared__ const float *rows[kTcTile];
    __shared__ float s_rew[kTcTile], s_done[kTcTile];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = warp & 3, half = warp >> 2;
    // trainer blockIdx.y of a grouped learner: its weight image, rows [r0, r0 + n) of the inputs / outputs, its keys
    const int grp = blockIdx.y;
    size_t r0 = (size_t)grp * (size_t)a.n;
    const unsigned char *img = a.img + (size_t)grp * (size_t)a.img_stride;
    // rows this grid row evaluates, tiles over them and the rows a tile advances by (LOSS: whole probe groups only)
    int n_rows = a.n, n_tiles = a.n_tiles, tile_step = a.rows_per_tile;
    int w_set = 0;
    if (LOSS) {
        w_set = a.loss_w0 + grp;
        const int lo = a.loss_tri ? 0 : kFedProbes * (w_set + 1), hi = a.loss_tri ? kFedProbes * w_set : a.n;
        r0 = (size_t)lo; n_rows = hi - lo;
        tile_step = (a.rows_per_tile / kFedProbes) * kFedProbes;
        n_tiles = (n_rows + tile_step - 1) / tile_step;
        img = a.img + (size_t)(w_set - a.loss_img0) * (size_t)a.img_stride;
        if ((int)blockIdx.x >= n_tiles) return;                  // nothing staged or waited for yet
    }
    // The first thread of the last warp initialises the two mbarriers and issues the weight copies while the other warps
    // already gather the first tile; the CTA-wide barrier in front of the first weight wait publishes the barriers.
    constexpr int kCtl = kTcThreads - 32;
    const bool early_w = (a.pdl & kPdlEarlyWeights) != 0;
    if (tid == kCtl) {
        mbar_init(&wbar, 1); mbar_init(&wbar2, 1); fence_barrier_init();
        if (early_w) stage_forward_image(tc, W, img, &wbar, &wbar2);
    }
    stage_trace(a.trace, 1);
    // PDL prologue (common.cuh): the weight image may be fetched before the wait when the predecessor does not write
    // it (TD passes after the env step); the first tile's rows may be gathered before the wait when the predecessor
    // does not write them (act after the optimiser kernel: observations were written two kernels back).
    bool waited = (a.pdl & kPdlEarlyRows) == 0;
    if (waited) {
        pdl_wait();
        pdl_trigger();
        if (tid == kCtl && !early_w) stage_forward_image(tc, W, img, &wbar, &wbar2);
    }

    // act mode: row b of the tile is simply obs[base + b] -- no replay sampling (Philox), no pointer table, no barrier
    constexpr bool direct = ACT;
    uint32_t pkey[4] = {0u, 0u, 0u, 0u};
    const BatchSrc src = direct ? a.src : trainer_src(a.src, grp, a.n, tc.in_dim);
    if (!direct) Philox::gen(src.key, src.epoch, 0x5A17ull, pkey);
    bool wready = false, w2ready = false;

    // R = real rows per tile (32 / 64 / 128, at most tc.max_rows).  A warpgroup's m64 MMA runs when its rows hold real
    // samples; accumulator rows >= R are computed from whatever SMEM follows the R-row operand (still inside this CTA's allocation) and never stored.
    // Small batches use R = 32 so that 4096 samples spread over 128 CTAs instead of 32.
    const int R = a.rows_per_tile;
    const EpiSlice e(R, kTcThreads);
    const int row = quad * 32 + lane;                            // the head epilogue's sample row (warps 0-3)
    const bool live = quad * 32 < R;                             // this warp's rows are real rows
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int base = tile * tile_step;
        if (!direct) {
            if (tid < R) {
                const int b = base + tid;
                const float *p = nullptr;
                float r = 0.f, d = 0.f;
                if (b < a.n) {
                    const Transition t = resolve_transition(src, b, tc.in_dim, pkey);
                    p = a.use_next ? t.s2 : t.s; r = t.r; d = t.d;
                }
                rows[tid] = p; s_rew[tid] = r; s_done[tid] = d;
            }
            __syncthreads();
        }
        stage_trace(a.trace, 27);
        a0_gather([&](int r) -> const float * {
            if (direct) return (base + r < n_rows && r < tile_step) ? a.obs + (r0 + base + r) * tc.in_dim : nullptr;
            return rows[r];
        }, R, tc.in_dim, tc.L[0].K_pad, Ahi, Alo);
        stage_trace(a.trace, 2);
        if (!waited) {
            pdl_wait();
            pdl_trigger();
            waited = true;
            if (tid == kCtl && !early_w) stage_forward_image(tc, W, img, &wbar, &wbar2);
        }
        if (!wready) {                                           // first tile: the control thread's barriers become visible
            __syncthreads();
            mbar_wait(&wbar, 0);
            wready = true;
        }
        stage_trace(a.trace, 3);
        fence_proxy_async();
        __syncthreads();
        stage_trace(a.trace, 4);

        const auto mid = [&](int l) {
            stage_trace(a.trace, 5 + 3 * l);
            if (!w2ready) { if (fwd_image_split(tc) < (uint32_t)tc.img_bytes) mbar_wait(&wbar2, 0); w2ready = true; }
            stage_trace(a.trace, 6 + 3 * l);
        };
        // head epilogue: Q row of this sample, then the mode's output
        const auto head = [&](int, const float *bias) {
            if (half == 0 && live) {
                const int nA = tc.n_actions;
                float q[32], bv;
                q_row<DUELING>(acc, tc.acc_ld, row, bias, nA, q);
                const int best = q_argmax(q, nA, bv);
                const int b = base + row;                               // trainer-local row
                const size_t ob = r0 + b;                               // its row in the [G][n] inputs / outputs
                if (LOSS) {
                    float d2 = 0.f;
                    if (b < n_rows && row < tile_step) {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < nA) { const float d = a.q_ref[ob * nA + j] - q[j]; d2 += d * d; }
                    }
                    s_rew[row] = d2;
                } else if (b < a.n) {
                    if (a.q_out) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < nA) a.q_out[ob * nA + j] = q[j];
                    }
                    if (ACT) {
                        int ra;
                        const bool greedy = eps_greedy(a.eps, a.is_train, a.u_tape, a.rand_tape, ob, trainer_key(a.key, kActSalt, grp), a.call, b, nA, ra);
                        a.actions[ob] = greedy ? best : ra;
                    } else if (!ACT && a.mode == kTcArgmax) {
                        a.actions[ob] = best;                                       // DDQN_Trainer.py:94
                    } else {                                                        // DQN_Trainer.py:109; DDQN_Trainer.py:95
                        const float nq = a.mode == kTcTdGather ? q_at(q, a.actions[ob]) : bv;
                        a.y_out[ob] = td_target(s_rew[row], a.gamma, nq, s_done[row]);
                    }
                }
            }
            __syncthreads();
            if (LOSS && tid * kFedProbes < tile_step && base + tid * kFedProbes < n_rows)   // one probe group per thread
                fed_group_loss(s_rew + tid * kFedProbes, r0 + base + tid * kFedProbes, a.loss_ld, w_set - a.loss_col0, tc.n_actions, a.loss_out);
        };
        forward_layers<FIXED, false>(tc, R, e, Ahi, Alo, W, acc, nullptr, false, mid, head,
                                     [&](int l, uint32_t) { stage_trace(a.trace, 7 + 3 * l); });
    }
    stage_trace(a.trace, 20);
}

template <bool ACT, bool DUELING, bool FIXED>
__global__ void __launch_bounds__(kTcThreads, 1) tc_forward_kernel_t(TcNet tc, TcArgs a)
{
    tc_forward_body<ACT, DUELING, FIXED, false>(tc, a);
}

template <bool DUELING, bool FIXED>
__global__ void __launch_bounds__(kTcThreads, 1) tc_loss_kernel_t(TcNet tc, TcArgs a)
{
    tc_forward_body<true, DUELING, FIXED, true>(tc, a);
}

bool tc_fixed_chains(const TcNet &tc, bool train)
{
    for (int l = 0; l < tc.n_layers; ++l) {
        const TcLayer &T = tc.L[l];
        if (!mma_fixed_product(kMmaFwd, T.N_pad, T.K_pad / 8)) return false;
        if (train && l > 0 && !mma_fixed_product(kMmaDx, T.K_pad, T.N_pad / 8)) return false;
    }
    return true;
}

typedef void (*ForwardKernel)(TcNet, TcArgs);
template <bool A, bool D>
static ForwardKernel pick_fwd_x(bool fixed) { return fixed ? tc_forward_kernel_t<A, D, true> : tc_forward_kernel_t<A, D, false>; }
template <bool A>
static ForwardKernel pick_fwd_d(bool dueling, bool fixed) { return dueling ? pick_fwd_x<A, true>(fixed) : pick_fwd_x<A, false>(fixed); }
static ForwardKernel pick_forward_kernel(bool act, bool dueling, bool fixed)
{
    return act ? pick_fwd_d<true>(dueling, fixed) : pick_fwd_d<false>(dueling, fixed);
}

template <bool D>
static ForwardKernel pick_loss_d(bool fixed) { return fixed ? tc_loss_kernel_t<D, true> : tc_loss_kernel_t<D, false>; }
static ForwardKernel pick_loss_kernel(bool dueling, bool fixed) { return dueling ? pick_loss_d<true>(fixed) : pick_loss_d<false>(fixed); }

int stage_trace_alloc(DevMem &m, long long *&t)
{
    static const bool on = getenv("UAVRL_TC_TRACE") != nullptr;
    t = nullptr;
    if (!on) return 0;
    return m.alloc(t, kTraceSlots);
}

int stage_trace_print(cudaStream_t st, const long long *t, const char *fmt, ...)
{
    if (!t) return 0;
    long long h[kTraceSlots];
    UAVRL_CUDA(cudaStreamSynchronize(st));
    UAVRL_CUDA(cudaMemcpy(h, t, sizeof(h), cudaMemcpyDeviceToHost));
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fprintf(stderr, " cycles since start:");
    for (int i = 1; i < kTraceSlots; ++i) if (h[i]) fprintf(stderr, " [%d]=%lld", i, h[i] - h[0]);
    fprintf(stderr, "\n");
    return 0;
}

int launch_tc_forward(uavrl_learner *l, const Route &r, const TcArgs &a_in, cudaStream_t st)
{
    TcArgs a = a_in;
    a.img_stride = l->tc.train_img_bytes;
    const int n_sm = num_sms();
    a.rows_per_tile = r.fwd_rows;
    a.n_tiles = (a.n + a.rows_per_tile - 1) / a.rows_per_tile;
    const int grid = a.n_tiles < n_sm ? a.n_tiles : n_sm;
    DevMem trace_mem;
    if (int rc = stage_trace_alloc(trace_mem, a.trace)) return rc;
    const ChainKernel kind = a.mode == kTcAct ? kChainAct : kChainTd;
    const ChainLaunch c = l->chain.next(kind);
    a.pdl = c.flags();
    UAVRL_CUDA(launch_kernel(pick_forward_kernel(a.mode == kTcAct, l->tc.dueling != 0, r.fwd == 2), dim3(grid, l->G), dim3(kTcThreads), tc_smem_bytes(l->tc), st, c.pdl, l->tc, a));
    l->chain.launched(kind);
    UAVRL_LAUNCHED();
    return stage_trace_print(st, a.trace, "[tc_trace] mode=%d n=%d R=%d grid=%d", a.mode, a.n, a.rows_per_tile, grid);
}

int launch_tc_loss(uavrl_learner *l, const Route &r, const TcArgs &a_in, int n_weights, int max_rows, cudaStream_t st)
{
    TcArgs a = a_in;
    a.img_stride = l->tc.train_img_bytes;
    a.rows_per_tile = r.fwd_rows;
    const int step = (a.rows_per_tile / kFedProbes) * kFedProbes;
    const int tiles = (max_rows + step - 1) / step, n_sm = num_sms();
    a.n_tiles = tiles;
    a.pdl = 0;
    UAVRL_CUDA(launch_kernel(pick_loss_kernel(l->tc.dueling != 0, r.fwd == 2), dim3(tiles < n_sm ? tiles : n_sm, n_weights),
                             dim3(kTcThreads), tc_smem_bytes(l->tc), st, false, l->tc, a));
    l->chain.launched(kChainNone);
    UAVRL_LAUNCHED();
    return 0;
}

int tc_init(uavrl_learner *l)
{
    std::vector<int32_t> hi, lo, hi2, lo2;
    l->tc_ok = false; l->tc_train_ok = false;
    if (tc_build(l->cfg, l->net, l->tc, hi, lo, hi2, lo2) != 0) return 0;
    l->tc_fixed_fwd = tc_fixed_chains(l->tc, false);
    l->tc_fixed_train = tc_fixed_chains(l->tc, true);
    const bool fixed = l->tc_fixed_fwd;
    size_t fwd_static = 0;                                       // the kernels' static shared memory (row table, barriers)
    for (int ac = 0; ac < 2; ++ac)
        for (int du = 0; du < 2; ++du) {
            cudaFuncAttributes fa;
            UAVRL_CUDA(cudaFuncGetAttributes(&fa, pick_forward_kernel(ac != 0, du != 0, fixed)));
            if (fa.sharedSizeBytes > fwd_static) fwd_static = fa.sharedSizeBytes;
        }
    if (tc_smem_bytes(l->tc) + fwd_static > kMaxBlockSmem) return 0;
    const size_t P = (size_t)l->net.P;
    const size_t img = (size_t)l->tc.train_img_bytes;
    const size_t img_all = (size_t)l->G * img;                  // [G] images of a grouped learner
    int rc;
    if ((rc = l->mem.alloc(l->tc_img_local, img_all)) || (rc = l->mem.alloc(l->tc_img_target, img_all))) return rc;
    int32_t **maps[] = { &l->tc_hi_map, &l->tc_lo_map, &l->tc_hi2_map, &l->tc_lo2_map };
    std::vector<int32_t> *src[] = { &hi, &lo, &hi2, &lo2 };
    for (int i = 0; i < 4; ++i) {
        if ((rc = l->mem.alloc(*maps[i], P, false))) return rc;
        UAVRL_CUDA(cudaMemcpy(*maps[i], src[i]->data(), P * 4, cudaMemcpyHostToDevice));
    }
    const size_t B = (size_t)l->G * l->cfg.batch_size;
    if ((rc = l->td_mem.alloc(l->y_buf, B, false)) || (rc = l->td_mem.alloc(l->astar_buf, B, false))) return rc;
    for (int ac = 0; ac < 2; ++ac)
        for (int du = 0; du < 2; ++du)
            if ((rc = raise_dyn_smem(pick_forward_kernel(ac != 0, du != 0, fixed), tc_smem_bytes(l->tc)))) return rc;
    for (int du = 0; du < 2; ++du)                               // the loss variant: the act kernel's static shared memory
        if ((rc = raise_dyn_smem(pick_loss_kernel(du != 0, fixed), tc_smem_bytes(l->tc)))) return rc;
    l->y_cap = l->cfg.batch_size;
    l->tc_ok = true;
    return tc_train_init(l);
}

}  // namespace uavrl
