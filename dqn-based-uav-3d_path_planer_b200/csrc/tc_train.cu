// tc_train.cu -- the TD update's forward + backward on the Hopper tensor cores (wgmma, 3xTF32), sm_90a.
//
// Replaces the arithmetic of Trainer.update (Trainer/DuelingDQN_Trainer.py:164-180, DDQN_Trainer.py:93-107,
// DQN_Trainer.py:107-126): Q(s).gather(a), MSE against the TD target, loss.backward().
//
//   tc_train_kernel  one CTA = R (32/64) sampled transitions.  The forward chain (tc_chain.cuh), then the
//                    loss / dLoss/dQ in the head epilogue, then the dX chain with the TRANSPOSED weight blocks of the
//                    training image:  dH_l = dZ_{l+1} * W_{l+1}  (A = dZ rows, B = W^T K-major), ReLU mask applied
//                    in the epilogue.  Hidden activations and every dZ are written once to a per-sample scratch
//                    (L2 resident: 4096 x ~0.9 KB) for the weight-gradient pass.
//   tc_dw_kernel     split-K weight gradients: CTA (layer l, chunk of 128 samples) computes
//                    dW_l^T [in+1 x out] = [act_l ; 1]^T (in+1 x 128) * dZ_l (128 x out)  -- the extra all-ones
//                    row yields the bias gradient for free -- and stores its slice of partial `chunk`.
//                    The contraction runs over SAMPLES while both operands are stored [sample][feature]: the rows are
//                    transposed into K-major operands on their way into SMEM (wgmma reads tf32 K-major only).
//                    reduce_adam_kernel then sums the partials.
// All products use the hi*hi + hi*lo + lo*hi TF32 split (fp32-grade, see tc_forward.cu).
#include <string.h>
#include <stdlib.h>

#include <atomic>

#include "tc_chain.cuh"

namespace uavrl {

constexpr int kDwChunk = 128;          // samples reduced by one dW CTA (the MMA's K extent)

struct TcTrainArgs {
    const unsigned char *img;          // local network, training image (forward blocks + biases + transposed blocks)
    BatchSrc src;
    int32_t B, R, n_tiles;
    const float *y;                    // [B] TD targets
    float inv_global_b;
    float *act_buf, *dz_buf;           // per-sample scratch rows
    float *loss_partials;              // [grid]
    int32_t loss_kind;                 // 0 MSE (reference), 1 Huber (delta = 1)
    // fused TD target (fused_td = 1; only when every CTA owns exactly one tile): the same CTA first evaluates the target
    // network (double DQN: the local network for a*, then the target network) on the tile's NEXT states and keeps
    // y = r + gamma * next_q * (1 - d) in shared memory -- one launch instead of two or three, no y round trip
    int32_t fused_td, algo;
    float gamma;
    const unsigned char *img_target;   // target network, forward image
    int64_t img_stride;                // grouped learner (gridDim.y = G): bytes between two trainers' images; y, the scratch rows
                                       // and the batch are [G][B], the loss partials [G][gridDim.x]
    long long *trace;                  // debug (UAVRL_TC_TRACE): CTA (0, 0) / thread 0 stage timestamps
};

struct TcDwArgs {
    BatchSrc src;
    int32_t B, n_chunks, P;
    int32_t n_slices;                  // CTAs per layer; slice i accumulates chunks i, i + n_slices, ... into partial i
    const float *act_buf, *dz_buf;
    float *partials;                   // [n_slices][P]
    long long *trace;                  // debug (UAVRL_TC_TRACE): CTA (0, 0) / thread 0 stage timestamps
};

// NPRE / DUELING are compile-time so that the kernel a configuration runs carries no code of the others: a third of the
// live warps' stall samples of the generic kernel were instruction-fetch stalls (143 KB of code, executed once per CTA).
// NPRE = forward-only TD passes ahead of the training chain (0: y comes from stand-alone passes, 1: DQN, 2: double DQN).
// FIXED: every layer product, forward and dX, is one unbroken compile-time wgmma chain (wgmma.cuh mma_fixed; tc_fixed_chains).
template <int NPRE, bool DUELING, bool FIXED>
__global__ void __launch_bounds__(kTcThreads, 1) tc_train_kernel(TcNet tc, TcTrainArgs a)
{
    stage_trace(a.trace, 0);
    extern __shared__ __align__(1024) unsigned char smem[];
    const int R = a.R;
    const uint32_t a_bytes = (uint32_t)(R / 8) * mma_sbo(tc.max_k);
    unsigned char *Ahi = smem, *Alo = smem + a_bytes, *W = smem + 2 * a_bytes;
    // R is 32 or 64: warpgroup 0's m64 MMA reads rows [R, 64) past the R-row operands (inside the allocation), never stored
    float *acc = reinterpret_cast<float *>(W + tc.train_img_bytes);     // accumulator tile [R][tc.acc_ld]
    __shared__ uint64_t wbar, wbar2, wbar3;                 // fused TD: training image in three pieces (below)
    __shared__ const float *rows[kTcTile];
    __shared__ const float *rows2[kTcTile];                  // fused TD: next-state rows
    __shared__ int s_act[kTcTile], s_astar[kTcTile];
    __shared__ uint8_t s_fresh[kTcTile];                     // fused TD: the next-state row is being written by this iteration's env step
    __shared__ float s_y[kTcTile], s_rew[kTcTile], s_done[kTcTile];
    __shared__ float s_loss[4];                              // per head warp, summed in warp order at the end: run-to-run exact

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = warp & 3, half = warp >> 2;
    // trainer blockIdx.y of a grouped learner: its images, batch, TD targets and scratch rows
    const int grp = blockIdx.y;
    const unsigned char *img = a.img + (size_t)grp * (size_t)a.img_stride, *img_t = a.img_target + (size_t)grp * (size_t)a.img_stride;
    const BatchSrc src = trainer_src(a.src, grp, a.B, tc.in_dim);
    const size_t r0 = (size_t)grp * (size_t)a.B;
    float *act_buf = a.act_buf + r0 * tc.act_stride, *dz_buf = a.dz_buf + r0 * tc.dz_stride;
    const float *y_in = a.y ? a.y + r0 : nullptr;
    // control thread (first of the last warp): barrier init and weight copies -- concurrently with warp 0 resolving the tile's
    // samples; the first CTA-wide barrier (behind the sample table) publishes the barriers
    constexpr int kCtl = kTcThreads - 32;
    if (tid == 0) s_loss[0] = s_loss[1] = s_loss[2] = s_loss[3] = 0.f;
    constexpr bool fused = NPRE > 0;
    constexpr int n_pre = NPRE;                                      // forward-only passes ahead of the training chain
    // PDL.  Unfused: the training image was written by the previous optimiser kernel (>= 2 kernels back: a TD pass always
    // precedes this kernel), so it is fetched before the wait, and so are the first tile's sampled rows and actions
    // (replay frames / actions were written by the env step and the act kernel, also >= 2 back); only y is the
    // predecessor's output.  Fused: the predecessor is the env step, which writes the newest frame's rows, rewards and
    // flags -- only the first pass's weight image (optimiser kernel, >= 2 back) is fetched before the wait.
    uint32_t wphase = 0;
    if (tid == kCtl) {
        mbar_init(&wbar, 1); mbar_init(&wbar2, 1); mbar_init(&wbar3, 1); fence_barrier_init();
        fence_proxy_async();
        if (!fused) bulk_g2s_chunked(W, img, (uint32_t)tc.train_img_bytes, &wbar);
        else {
            bulk_g2s_chunked(W, (n_pre == 2) ? img : img_t, (uint32_t)tc.img_bytes, &wbar);
            // the transposed blocks of the training image (dX chain) lie behind the forward image the TD passes use: they are
            // fetched now (written by the optimiser step, >= 2 kernels back) and first waited for in front of the dX chain
            if (tc.train_img_bytes > tc.img_bytes)
                bulk_g2s_chunked(W + tc.img_bytes, img + tc.img_bytes, (uint32_t)(tc.train_img_bytes - tc.img_bytes), &wbar3);
        }
    }
    stage_trace(a.trace, 1);
    bool waited = false;

    uint32_t pkey[4];
    Philox::gen(src.key, src.epoch, 0x5A17ull, pkey);
    bool wready = false;
    const int nl = tc.n_layers;
    const int row = quad * 32 + lane;                        // the head epilogues: one sample row per thread of warps 0-3
    const bool live = quad * 32 < R;
    // the hidden-layer and dX epilogues run on every thread: row e.row, 4-column groups e.c0 + i * e.step (i = 0, 1, ...)
    const EpiSlice e(R, kTcThreads);
    // ReLU' for the dX chain: bit 4i + j of hmK = (H_K[e.row][e.c0 + i * e.step + j] > 0), kept from the forward epilogue of the
    // same thread (hidden layers are at most 64 wide and R <= 64 here: at most 16 elements per thread) -- no reload of H
    uint32_t hm1 = 0u, hm2 = 0u, hm3 = 0u, hm4 = 0u;
    const auto table = [](const float *const *t) { return [t](int r) { return t[r]; }; };

    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int base = tile * R;
        // where the tile's rows are: index arithmetic only (resolve_rows), so with the fused TD pass it runs BEFORE the wait for
        // the env step; the transitions' action / reward / done are requested right after the wait and parked in shared memory
        // once the first gather has been issued (they are first read in a head epilogue)
        int64_t my_slot = -1;
        if (tid < R) {
            const int b = base + tid;
            const float *p = nullptr, *p2 = nullptr;
            bool fr = false;
            if (b < a.B) my_slot = resolve_rows(src, b, tc.in_dim, pkey, p, p2, &fr);
            rows[tid] = p;
            if (fused) { rows2[tid] = p2; s_astar[tid] = 0; s_fresh[tid] = fr ? 1 : 0; }
        }
        __syncthreads();                                         // the sample table -- and, first time round, the barriers
        // Fused TD (one tile per CTA, at most 4 items per thread): BOTH gathers are requested before the wait for the env step --
        // the training rows (never younger than the previous iteration) and every next-state row outside the frame that env step
        // is writing (all but ~N/count of them); the few fresh ones follow after the wait from L2.  The HBM latency of the
        // sampled rows is then hidden behind the predecessor instead of heading this kernel's chain.
        const bool early_rows = n_pre > 0 && R * (tc.L[0].K_pad / 4) <= 4 * kTcThreads;
        float4 vmain[4], vnext[4];
        if (early_rows) {
            a0_load_sel(rows2, s_fresh, false, R, tc.in_dim, tc.L[0].K_pad, vnext);
            a0_load(table(rows), tid, R, tc.in_dim, tc.L[0].K_pad, vmain);
        }
        if (fused && !waited) { pdl_wait(); pdl_trigger(); waited = true; }
        int m_act = 0; float m_rew = 0.f, m_done = 0.f;
        if (my_slot >= 0) load_meta(src, my_slot, m_act, m_rew, m_done);
        if (early_rows) a0_load_sel(rows2, s_fresh, true, R, tc.in_dim, tc.L[0].K_pad, vnext);
        auto park_meta = [&]() { if (tid < R) { s_act[tid] = m_act; if (fused) { s_rew[tid] = m_rew; s_done[tid] = m_done; } } };
        stage_trace(a.trace, 2);
        // ---------------- fused TD target: forward-only pass(es) on the next states
        for (int pass = 0; pass < n_pre; ++pass) {
            if (pass > 0 && tid == kCtl) {                                     // the target image replaces the local one (all its readers are done)
                fence_proxy_async();
                bulk_g2s_chunked(W, img_t, (uint32_t)tc.img_bytes, &wbar);
            }
            if (pass == 0 && early_rows) a0_store(vnext, tid, R, tc.L[0].K_pad, Ahi, Alo);
            else a0_gather(table(rows2), R, tc.in_dim, tc.L[0].K_pad, Ahi, Alo);
            if (pass == 0) { park_meta(); stage_trace(a.trace, 3); }
            mbar_wait(&wbar, wphase); wphase ^= 1;
            fence_proxy_async();
            __syncthreads();
            if (pass == 0) stage_trace(a.trace, 4);
            const bool td_pass = (pass == n_pre - 1);
            const auto head = [&](int l, const float *bias) {
                if (half == 0 && live) {
                    float q[32], bv;
                    q_row<DUELING>(acc, tc.acc_ld, row, bias, tc.n_actions, q);
                    const int best = q_argmax(q, tc.n_actions, bv);
                    if (!td_pass) s_astar[row] = best;                                  // DDQN_Trainer.py:94
                    else s_y[row] = td_target(s_rew[row], a.gamma, n_pre == 2 ? q_at(q, s_astar[row]) : bv, s_done[row]);  // DDQN_Trainer.py:95
                }
                fence_proxy_async();
                __syncthreads();
                if (pass == 0) stage_trace(a.trace, 5 + l);
            };
            forward_layers<FIXED, false>(tc, R, e, Ahi, Alo, W, acc, nullptr, false, [](int) {}, head,
                                         [&](int l, uint32_t) { if (pass == 0) stage_trace(a.trace, 5 + l); });
        }
        if (fused && tid == kCtl) stage_forward_image(tc, W, img, &wbar, &wbar2);     // the training image (every reader of the TD image is done)
        if (early_rows) a0_store(vmain, tid, R, tc.L[0].K_pad, Ahi, Alo);
        else a0_gather(table(rows), R, tc.in_dim, tc.L[0].K_pad, Ahi, Alo);
        stage_trace(a.trace, 9);
        if (!waited) { pdl_wait(); pdl_trigger(); waited = true; }
        if (n_pre == 0) park_meta();
        if (!fused && tid < R) s_y[tid] = (base + tid < a.B) ? y_in[base + tid] : 0.f;      // visible after the barrier below
        if (fused) { mbar_wait(&wbar, wphase); wphase ^= 1; }
        else if (!wready) { mbar_wait(&wbar, 0); wready = true; }
        fence_proxy_async();
        __syncthreads();
        stage_trace(a.trace, 10);
        const int gb = base + row;                          // this thread's sample in the head epilogue (valid when live && gb < B)
        const bool mine = live && gb < a.B;
        const int egb = base + e.row;                       // ... and in the hidden-layer / dX epilogues
        const bool emine = egb < a.B;

        // ---------------- forward chain: activations kept for dW, ReLU masks for the dX chain
        const auto mid = [&](int l) {
            if (fused && l == 0 && fwd_image_split(tc) < (uint32_t)tc.img_bytes) mbar_wait(&wbar2, 0);     // biases + the later layers' weights
            if (l < 4) stage_trace(a.trace, 27 + l);
        };
        // head: Q(s, .), loss, dLoss/dHead -> next A operand (K = 32) and the dz scratch
        const auto head = [&](int l, const float *bias) {
            const TcLayer &T = tc.L[l];
            if (half == 0 && live) {
                const int nA = tc.n_actions;
                float q[32];
                acc_ld32(acc, tc.acc_ld, row, 0, q);
                stage_trace(a.trace, 21);
                q_combine<DUELING>(bias, nA, q);
                const int act = s_act[row];
                const float qa = q_at(q, act);
                stage_trace(a.trace, 22);
                float gq = 0.f, lterm = 0.f;
                if (mine) lterm = td_loss(src, gb, qa - s_y[row], a.loss_kind, a.inv_global_b, gq);
                // the warp's 32 loss terms: butterfly sum, then one add into the warp's own shared word.  A shared atomicAdd of
                // every head warp into one word summed the warps in arrival order, so a CTA with two 64-row tiles reported a
                // loss that could differ by an ulp from run to run
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) lterm += __shfl_xor_sync(0xffffffffu, lterm, off);
                stage_trace(a.trace, 23);
                if (lane == 0) s_loss[quad] += lterm;
                stage_trace(a.trace, 24);
                float g[32];
                const float inv = 1.f / (float)nA;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    float gj;
                    if (DUELING) gj = (j < nA) ? gq * ((j == act ? 1.f : 0.f) - inv) : (j == nA ? gq : 0.f);
                    else gj = (j == act) ? gq : 0.f;
                    g[j] = gj;
                }
                stage_trace(a.trace, 25);
                const uint32_t sbon = mma_sbo(T.N_pad);
                float *dz_row = dz_buf + (size_t)gb * tc.dz_stride + T.dz_off;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float4 x = make_float4(g[4 * j], g[4 * j + 1], g[4 * j + 2], g[4 * j + 3]), h, lo4;
                    tf32_split(x.x, h.x, lo4.x); tf32_split(x.y, h.y, lo4.y); tf32_split(x.z, h.z, lo4.z); tf32_split(x.w, h.w, lo4.w);
                    const uint32_t off = mma_off(row, 4 * j, sbon);
                    *reinterpret_cast<float4 *>(Ahi + off) = h;
                    *reinterpret_cast<float4 *>(Alo + off) = lo4;
                    if (mine) *reinterpret_cast<float4 *>(dz_row + 4 * j) = x;
                }
                stage_trace(a.trace, 26);
            }
            fence_proxy_async();
            __syncthreads();
            stage_trace(a.trace, 11 + l);
        };
        forward_layers<FIXED, true>(tc, R, e, Ahi, Alo, W, acc, act_buf + (size_t)egb * tc.act_stride, emine, mid, head,
                                    [&](int l, uint32_t mk) {
                                        if (l == 0) hm1 = mk; else if (l == 1) hm2 = mk; else if (l == 2) hm3 = mk; else hm4 = mk;
                                        stage_trace(a.trace, 11 + l);
                                    });

        if (fused && tc.train_img_bytes > tc.img_bytes) mbar_wait(&wbar3, 0);                     // transposed blocks (requested at kernel start)
        // ---------------- dX chain: dZ_{l-1} = (dZ_l * W_l) .* (H_l > 0), l = nl-1 .. 1
        for (int l = nl - 1; l >= 1; --l) {
            const TcLayer T = tc.L[l];
            mma_3xtf32<kMmaDx, FIXED>(acc, tc.acc_ld, Ahi, Alo, W + T.t_hi_off, W + T.t_lo_off, mma_sbo(T.N_pad), T.K_pad, T.N_pad / 8, R);
            // ReLU'(H_l): the sign mask this thread kept in the forward epilogue of the same columns (K_pad(l) = N_pad(l - 1))
            const uint32_t hmask = (l == 1) ? hm1 : (l == 2) ? hm2 : (l == 3) ? hm3 : hm4;
            const uint32_t sbon = mma_sbo(T.K_pad);
            float *dz_row = dz_buf + (size_t)egb * tc.dz_stride + tc.L[l - 1].dz_off;
            for (int c = e.c0, sh = 0; c < T.K_pad; c += e.step, sh += 4) {
                const float4 v = e.ld(acc, tc.acc_ld, c);
                const uint32_t m4 = hmask >> sh;
                float4 x, h, lo4;
                x.x = (m4 & 1u) ? v.x : 0.f; x.y = (m4 & 2u) ? v.y : 0.f;
                x.z = (m4 & 4u) ? v.z : 0.f; x.w = (m4 & 8u) ? v.w : 0.f;
                if (emine) *reinterpret_cast<float4 *>(dz_row + c) = x;
                if (l > 1) {
                    tf32_split(x.x, h.x, lo4.x); tf32_split(x.y, h.y, lo4.y); tf32_split(x.z, h.z, lo4.z); tf32_split(x.w, h.w, lo4.w);
                    const uint32_t off = mma_off(e.row, c, sbon);
                    *reinterpret_cast<float4 *>(Ahi + off) = h;
                    *reinterpret_cast<float4 *>(Alo + off) = lo4;
                }
            }
            fence_proxy_async();
            __syncthreads();
            stage_trace(a.trace, 16 + l);
        }
    }
    stage_trace(a.trace, 20);
    // the head epilogue ends with a CTA barrier: every warp's last add is visible here
    if (tid == 0) a.loss_partials[(size_t)grp * gridDim.x + blockIdx.x] = ((s_loss[0] + s_loss[1]) + s_loss[2]) + s_loss[3];
}

// ------------------------------------------------------------------ split-K weight gradients
// Both products contract over the chunk's 128 samples, and wgmma reads tf32 operands K-major only: the rows ([sample][feature]
// in global memory) are transposed on their way into shared memory, element (feature f, sample b) of a [features][128 samples]
// K-major operand.  The SBO carries 16 bytes of padding so that a warp's scalar stores (one sample, 128 consecutive features)
// spread over 8 banks instead of 2.
constexpr uint32_t kDwSbo = (kDwChunk / 4) * 128u + 16u;   // bytes per 8-feature group: 128 samples x 4 B x 8 (+ 16)
constexpr int kDwARows = 128;                               // A operand: input features + the ones column, zero padded

// rows [128 samples][width floats] in global memory -> hi/lo K-major operands.  8 consecutive lanes load one 128-byte
// row segment (coalesced).
// LOG2F4 = log2(float4 per row) (5 for the 128-wide A operand, 3 / 4 for a 32- / 64-wide B operand); U float4 per thread,
// ALL loaded before the first is converted (the loads are the latency that matters: one round trip per operand).
// ones_col >= 0: that feature column is set to 1 for valid samples (bias gradient).
template <int LOG2F4, int U>
__device__ __forceinline__ void dw_load_rows(const float *const *rows, int width, float4 (&v)[U])
{
    // nothing but loads here: a register that a load is still going to write must not be touched again before the data
    // is consumed, or the warp stalls on that load before issuing the next one (the ones column is applied at store time)
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int i = threadIdx.x + u * kTcThreads;
        const int b = i >> LOG2F4, jc = i & ((1 << LOG2F4) - 1);
        const float *r = (b < kDwChunk) ? rows[b] : nullptr;
        v[u] = (r && 4 * jc < width) ? __ldg(reinterpret_cast<const float4 *>(r) + jc) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}
// ones_col >= 0: that feature column (a multiple of 4: K_real % 4 == 0, tc_train_init) becomes 1 for valid samples
template <int LOG2F4, int U>
__device__ __forceinline__ void dw_store_rows(const float4 (&v)[U], const float *const *rows, int ones_col, unsigned char *hi, unsigned char *lo)
{
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int i = threadIdx.x + u * kTcThreads;
        const int b = i >> LOG2F4, jc = i & ((1 << LOG2F4) - 1);
        if (b >= kDwChunk) continue;
        float4 x = v[u];
        if (ones_col >= 0 && (ones_col >> 2) == jc && rows[b]) x.x = 1.f;
        const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float h, l;
            tf32_split(xs[e], h, l);
            const uint32_t off = mma_off(4 * jc + e, b, kDwSbo);
            *reinterpret_cast<float *>(hi + off) = h;
            *reinterpret_cast<float *>(lo + off) = l;
        }
    }
}

__global__ void __launch_bounds__(kTcThreads, 1) tc_dw_kernel(TcNet tc, TcDwArgs a)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const int l = blockIdx.x % tc.n_layers, slice = blockIdx.x / tc.n_layers;
    const int chunk = slice;                                  // partial index
    // trainer blockIdx.y of a grouped learner: its batch, scratch rows and partials [n_slices][P]
    const int grp = blockIdx.y;
    const BatchSrc src = trainer_src(a.src, grp, a.B, tc.in_dim);
    const float *act_buf = a.act_buf + (size_t)grp * a.B * tc.act_stride, *dz_buf = a.dz_buf + (size_t)grp * a.B * tc.dz_stride;
    const TcLayer T = tc.L[l];
    const int rowsA = T.K_real + 1;                           // input features + the all-ones column (bias gradient)
    // A = [act ; 1]^T as [feature][sample] (rows past rowsA are zero), B = dZ^T as [out][sample]; hi and lo images of each
    unsigned char *Ahi = smem, *Alo = Ahi + (kDwARows / 8) * kDwSbo, *Bhi = Alo + (kDwARows / 8) * kDwSbo;
    unsigned char *Blo = Bhi + (T.N_pad / 8) * kDwSbo;
    __shared__ const float *rows[2][kDwChunk];               // double buffered: chunk c + 1 is resolved while chunk c is loaded
    __shared__ const float *drows[2][kDwChunk];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = warp & 3, half = warp >> 2;
    stage_trace(a.trace, 0);
    uint32_t pkey[4];
    Philox::gen(src.key, src.epoch, 0x5A17ull, pkey);
    auto resolve_chunk = [&](int c, int buf) {                // row pointers of chunk c (128 samples)
        if (tid < kDwChunk) {
            const int b = c * kDwChunk + tid;
            const float *p = nullptr, *dzp = nullptr;
            if (c < a.n_chunks && b < a.B) {
                p = (l == 0) ? resolve_transition(src, b, tc.in_dim, pkey).s : act_buf + (size_t)b * tc.act_stride + T.act_off;
                dzp = dz_buf + (size_t)b * tc.dz_stride + T.dz_off;
            }
            rows[buf][tid] = p; drows[buf][tid] = dzp;
        }
    };
    resolve_chunk(slice, 0);
    __syncthreads();
    // PDL: hidden activations and dZ come from the training chain (the predecessor); the layer-0 CTAs' A operand is
    // built from replay rows (written >= 2 kernels back) and is gathered before the wait
    if (l != 0) { pdl_wait(); pdl_trigger(); }
    stage_trace(a.trace, 1);
    // A: 128 samples x 128 columns (features, the ones column, zero padding) = 16 float4 per thread; B: 128 x N_pad.
    // Persistent over this slice's chunks: the loads of chunk c + 1 are issued before the MMAs of chunk c and land while they
    // run; the products accumulate in the same registers -> one partial per slice however large the batch.
    float4 va[16], vb[8];
    auto load_chunk = [&](int buf) {
        dw_load_rows<5, 16>(rows[buf], T.K_real, va);
        if (T.N_pad == 32) {
#pragma unroll
            for (int u = 4; u < 8; ++u) vb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            dw_load_rows<3, 4>(drows[buf], 32, reinterpret_cast<float4 (&)[4]>(vb));
        } else {
            dw_load_rows<4, 8>(drows[buf], 64, vb);         // N_pad = 64
        }
    };
    if (l == 0) {                                              // replay rows first, dZ after the predecessor has finished
        dw_load_rows<5, 16>(rows[0], T.K_real, va);
        pdl_wait(); pdl_trigger();
        if (T.N_pad == 32) {
#pragma unroll
            for (int u = 4; u < 8; ++u) vb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            dw_load_rows<3, 4>(drows[0], 32, reinterpret_cast<float4 (&)[4]>(vb));
        } else {
            dw_load_rows<4, 8>(drows[0], 64, vb);
        }
    } else {
        load_chunk(0);
    }
    stage_trace(a.trace, 2);
    // warpgroup g owns features [64g, 64g + 64); its MMAs run when that range holds real rows
    const int row0 = (tid >> 7) * 64;
    const bool wg_live = row0 < rowsA;
    float d[32];
    int it = 0;
    for (int c = slice; c < a.n_chunks; c += a.n_slices, ++it) {
        if (it > 0) __syncthreads();                           // both warpgroups' MMAs of the previous chunk have read SMEM
        dw_store_rows<5, 16>(va, rows[it & 1], T.K_real, Ahi, Alo);
        if (T.N_pad == 32) dw_store_rows<3, 4>(reinterpret_cast<float4 (&)[4]>(vb), drows[it & 1], -1, Bhi, Blo);
        else dw_store_rows<4, 8>(vb, drows[it & 1], -1, Bhi, Blo);
        const int cn = c + a.n_slices;
        resolve_chunk(cn, (it + 1) & 1);
        fence_proxy_async();
        __syncthreads();
        stage_trace(a.trace, 4);
        if (cn < a.n_chunks) load_chunk((it + 1) & 1);         // next chunk's rows -> registers while the MMAs run
        if (wg_live) {
            const uint64_t ah = mma_desc(Ahi + (row0 / 8) * kDwSbo, kDwSbo), al = mma_desc(Alo + (row0 / 8) * kDwSbo, kDwSbo);
            const uint64_t bh = mma_desc(Bhi, kDwSbo), bl = mma_desc(Blo, kDwSbo);
            if (T.N_pad == 32) wgmma_3xtf32<32>(d, ah, al, bh, bl, kDwChunk / 8, it > 0 ? 1u : 0u);
            else wgmma_3xtf32<64>(d, ah, al, bh, bl, kDwChunk / 8, it > 0 ? 1u : 0u);
        }
    }
    stage_trace(a.trace, 5);
    // the accumulator -> a [feature][out] tile in the A operand's space (every MMA has read it), one feature row per thread
    __syncthreads();
    float *acc = reinterpret_cast<float *>(smem);
    const int acc_ld = T.N_pad + 4;
    if (wg_live) {
        if (T.N_pad == 32) store_frag<32>(d, acc, acc_ld, row0, 0, kDwARows);
        else store_frag<64>(d, acc, acc_ld, row0, 0, kDwARows);
    }
    __syncthreads();
    stage_trace(a.trace, 6);
    // epilogue: row f = input feature (or the ones column), column o = output unit, into partial slice `chunk`.
    // Lanes hold consecutive f, so every store instruction writes 32 consecutive elements of one weight row; the 32 columns of a
    // thread walk the rows with a pointer increment and a predicate each (the address arithmetic used to dominate this epilogue).
    float *part = a.partials + ((size_t)grp * a.n_slices + chunk) * a.P;
    const int f = quad * 32 + lane;
    for (int c0 = half * 32; c0 < T.N_pad; c0 += 64) {
        if (quad * 32 >= rowsA) break;
        float v[32];
        acc_ld32(acc, acc_ld, f, c0, v);
        const int n_main = min(max(T.out_main - c0, 0), 32), n_all = min(max(T.N_real - c0, 0), 32);   // columns [0, n_main): main block, [n_main, n_all): value head
        if (f > T.K_real) continue;
        const bool brow = (f == T.K_real);                       // the ones column: bias gradients (stride 1), else weight row f (stride K_real)
        const int stride = brow ? 1 : T.K_real;
        const int i_main = brow ? T.b_off + c0 : T.w_off + f + c0 * T.K_real;
        const int i_val = brow ? T.b2_off + (c0 - T.out_main) : (T.w2_off >= 0 ? T.w2_off : 0) + f + (c0 - T.out_main) * T.K_real;
        float *p = part + i_main;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            if (j < n_main) *p = v[j];
            p += stride;
        }
        if (n_all > n_main) {
            float *q = part + i_val;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                if (j >= n_main && j < n_all) *q = v[j];
                q += stride;
            }
        }
    }
    stage_trace(a.trace, 7);
}

typedef void (*TrainKernel)(TcNet, TcTrainArgs);
template <int N, bool D>
static TrainKernel pick_train_x(bool fixed) { return fixed ? tc_train_kernel<N, D, true> : tc_train_kernel<N, D, false>; }
template <int N>
static TrainKernel pick_train_d(bool dueling, bool fixed) { return dueling ? pick_train_x<N, true>(fixed) : pick_train_x<N, false>(fixed); }
static TrainKernel pick_train_kernel(int npre, bool dueling, bool fixed)
{
    return npre == 0 ? pick_train_d<0>(dueling, fixed) : npre == 1 ? pick_train_d<1>(dueling, fixed) : pick_train_d<2>(dueling, fixed);
}

static size_t train_smem_bytes(const TcNet &tc, int R)
{
    return (size_t)2 * (R / 8) * mma_sbo(tc.max_k) + (size_t)tc.train_img_bytes + (size_t)R * tc.acc_ld * 4;   // + the accumulator tile
}
static size_t dw_smem_bytes(const TcNet &tc)
{
    int maxN = 32;
    for (int l = 0; l < tc.n_layers; ++l) if (tc.L[l].N_pad > maxN) maxN = tc.L[l].N_pad;
    return (size_t)2 * ((kDwARows + maxN) / 8) * kDwSbo;        // A hi/lo + B hi/lo
}

int tc_train_init(uavrl_learner *l)
{
    l->tc_train_ok = false;
    TcNet &tc = l->tc;
    tc.train_max_rows = 0;
    for (int i = 0; i < tc.n_layers; ++i)
        if (tc.L[i].K_real + 1 > 128 || tc.L[i].K_real % 4 != 0 || (tc.L[i].N_pad != 32 && tc.L[i].N_pad != 64)) return 0;   // ones column / float4 chunks / 1-2 blocks
    // a block's 227 KB hold the kernels' static shared memory (sample tables, barriers) as well as the dynamic allocation
    const bool fixed = tc_fixed_chains(tc, true);
    size_t train_static = 0, dw_static = 0;
    for (int np = 0; np < 3; ++np)
        for (int du = 0; du < 2; ++du) {
            cudaFuncAttributes fa;
            UAVRL_CUDA(cudaFuncGetAttributes(&fa, pick_train_kernel(np, du != 0, fixed)));
            if (fa.sharedSizeBytes > train_static) train_static = fa.sharedSizeBytes;
        }
    {
        cudaFuncAttributes fa;
        UAVRL_CUDA(cudaFuncGetAttributes(&fa, tc_dw_kernel));
        dw_static = fa.sharedSizeBytes;
    }
    const size_t train_budget = (size_t)227 * 1024 - train_static;
    // the m64 MMA reads 8 row groups from each A buffer: with fewer real rows it runs into the next buffers,
    // which must still be inside the CTA's allocation
    if (train_smem_bytes(tc, 32) > train_budget || dw_smem_bytes(tc) + dw_static > (size_t)227 * 1024) return 0;
    if (train_smem_bytes(tc, 32) < (size_t)(32 / 8) * mma_sbo(tc.max_k) + (size_t)8 * mma_sbo(tc.max_k)) return 0;
    tc.train_max_rows = train_smem_bytes(tc, 64) <= train_budget ? 64 : 32;
    for (int np = 0; np < 3; ++np)
        for (int du = 0; du < 2; ++du)
            if (int rc = raise_dyn_smem(pick_train_kernel(np, du != 0, fixed), train_smem_bytes(tc, tc.train_max_rows))) return rc;
    if (int rc = raise_dyn_smem(tc_dw_kernel, dw_smem_bytes(tc))) return rc;
    const size_t cap = (size_t)l->cfg.batch_size, G = (size_t)l->G;
    UAVRL_CUDA(cudaMalloc((void **)&l->act_buf, G * cap * (size_t)(tc.act_stride > 0 ? tc.act_stride : 4) * 4));
    UAVRL_CUDA(cudaMalloc((void **)&l->dz_buf, G * cap * (size_t)tc.dz_stride * 4));
    l->train_cap = (int32_t)cap;
    l->tc_train_ok = true;
    return 0;
}

std::atomic<int> g_fuse_td{1};               // uavrl_set_fuse_td(); default on
// rows per tile of the training kernel: 32 while the batch fits one wave of 32-row tiles, else 64 (when the 64-row operands fit)
int train_rows_per_tile(const TcNet &tc, int B)
{
    return (B > 32 * num_sms() && tc.train_max_rows == 64) ? 64 : 32;
}
bool tc_train_can_fuse_td(const uavrl_learner *l, int B)
{
    // one tile per CTA (32-row tiles up to 4 736 samples, 64-row tiles up to 9 472): the weight images are restaged inside the
    // kernel, which only pays when a CTA does it once; larger batches keep the separate TD-target kernel(s) whose CTAs reuse
    // one image over several tiles
    if (!g_fuse_td.load() || !l->tc_train_ok) return false;
    const int R = train_rows_per_tile(l->tc, B);
    return (B + R - 1) / R <= num_sms();
}
int launch_tc_train(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, const float *y, int *n_grad_parts,
                    int *n_loss_parts, cudaStream_t st, cudaEvent_t after_chain, bool fused_td)
{
    const TcNet &tc = l->tc;
    TcTrainArgs a;
    memset(&a, 0, sizeof(a));
    a.img = l->tc_img_local; a.src = src; a.B = B; a.y = y; a.inv_global_b = 1.0f / (float)global_batch;
    a.act_buf = l->act_buf; a.dz_buf = l->dz_buf; a.loss_partials = l->loss_partials;
    a.loss_kind = l->cfg.loss_kind;
    a.fused_td = fused_td ? 1 : 0; a.algo = l->cfg.algo; a.gamma = l->cfg.gamma; a.img_target = l->tc_img_target;
    a.img_stride = tc.train_img_bytes;
    a.R = train_rows_per_tile(tc, B);
    a.n_tiles = (B + a.R - 1) / a.R;
    const int grid = a.n_tiles < num_sms() ? a.n_tiles : num_sms();
    const bool chain = l->pdl_chain && g_pdl.load();
    if (fused_td && a.n_tiles > grid) return fail(UAVRL_ERR_INVALID, "fused TD needs one tile per CTA");
    TcDwArgs d;
    memset(&d, 0, sizeof(d));
    if (int rc = stage_trace_alloc(&a.trace)) return rc;
    if (int rc = stage_trace_alloc(&d.trace)) { cudaFree(a.trace); return rc; }
    const bool use_pdl = chain && (fused_td ? (l->pdl_prev == kPdlEnv) : (l->pdl_prev == kPdlTd));
    const int npre = fused_td ? (l->cfg.algo != UAVRL_ALGO_DQN ? 2 : 1) : 0;
    UAVRL_CUDA(launch_kernel(pick_train_kernel(npre, tc.dueling != 0, tc_fixed_chains(tc, true)), dim3(grid, l->G), dim3(kTcThreads),
                             train_smem_bytes(tc, a.R), st, use_pdl, tc, a));
    l->pdl_prev = chain ? kPdlTrain : kPdlNone;
    UAVRL_LAUNCHED();
    if (after_chain) UAVRL_CUDA(cudaEventRecord(after_chain, st));
    d.src = src; d.B = B; d.n_chunks = (B + kDwChunk - 1) / kDwChunk; d.P = l->net.P;
    d.act_buf = l->act_buf; d.dz_buf = l->dz_buf; d.partials = l->partials;
    const int n_sm = num_sms();
    // one CTA per SM (193 KB of shared memory): at most n_sm / n_layers slices per layer, each looping over its chunks
    const int max_slices = n_sm / tc.n_layers > 0 ? n_sm / tc.n_layers : 1;
    d.n_slices = d.n_chunks < max_slices ? d.n_chunks : max_slices;
    const int dw_grid = d.n_slices * tc.n_layers;
    UAVRL_CUDA(launch_kernel(tc_dw_kernel, dim3(dw_grid, l->G), dim3(kTcThreads), dw_smem_bytes(tc), st, chain && !after_chain, tc, d));
    l->pdl_prev = chain ? kPdlDw : kPdlNone;
    UAVRL_LAUNCHED();
    const int rc_train = stage_trace_print(st, a.trace, "[train_trace] B=%d R=%d fused_td=%d", B, a.R, a.fused_td);
    const int rc_dw = stage_trace_print(st, d.trace, "[dw_trace] B=%d chunks=%d (CTA 0 = layer 0)", B, d.n_chunks);     // frees d.trace either way
    if (rc_train || rc_dw) return rc_train ? rc_train : rc_dw;
    *n_grad_parts = d.n_slices;
    *n_loss_parts = grid;
    return 0;
}

}  // namespace uavrl

// kept for ABI compatibility: the optimiser step always runs as its own kernel
extern "C" int uavrl_set_fuse_dw_adam(int32_t on)
{
    return on ? uavrl::fail(UAVRL_ERR_INVALID, "uavrl_set_fuse_dw_adam: the fused weight-gradient + optimiser variant was removed") : 0;
}
extern "C" int uavrl_set_fuse_td(int32_t on) { uavrl::g_fuse_td.store(on ? 1 : 0); return 0; }
extern "C" int uavrl_learner_td_fused(const uavrl_learner *l, int32_t batch) { return (l && l->tc_ok && l->use_tc && uavrl::tc_train_can_fuse_td(l, batch)) ? 1 : 0; }
// the same decisions launch_act / launch_update_impl take (uavrl.h)
extern "C" int uavrl_learner_tc_route(const uavrl_learner *l, int32_t n, int32_t *out)
{
    if (!l || !out || n <= 0) return uavrl::fail(UAVRL_ERR_INVALID, "bad argument");
    const bool fwd = l->tc_ok && l->use_tc, train = fwd && l->tc_train_ok;
    out[0] = fwd ? (uavrl::tc_fixed_chains(l->tc, false) ? 2 : 1) : 0;
    out[1] = train ? (uavrl::tc_fixed_chains(l->tc, true) ? 2 : 1) : 0;
    out[2] = fwd ? uavrl::tc_forward_rows_per_tile(l->tc, n) : 0;
    out[3] = train ? uavrl::train_rows_per_tile(l->tc, n) : 0;
    out[4] = (train && uavrl::tc_train_can_fuse_td(l, n)) ? 1 : 0;
    out[5] = l->dual_weights;
    return 0;
}
