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
// forms Q (dueling combine), then eps-greedy / argmax / max / gather depending on the mode.
#include "tc_forward.cuh"
#include "env_block.cuh"

#include <stdlib.h>
#include <string.h>

#include "tma.cuh"
#include "wgmma.cuh"

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
    if (tc_smem_bytes(tc) + 4096 > 227 * 1024) {                 // 128 rows of operands + accumulator, weights, static smem
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


#define TC_TRACE(slot) do { if (a.trace && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) a.trace[slot] = clock64(); } while (0)

// FUSE_ENV: after a tile's actions are written, the same CTA steps those R envs (env_block.cuh) -- the act -> step
// dependency is per env, so no grid-wide boundary is needed between Trainer.get_action and BaseEnv.Move_Agent.
// ACT (a.mode == kTcAct) and DUELING are compile-time: the kernel a pass runs carries no code of the other modes.
// FIXED: every layer product is one unbroken compile-time wgmma chain (wgmma.cuh mma_fixed; tc_fixed_chains).
template <bool FUSE_ENV, bool ACT, bool DUELING, bool FIXED>
__global__ void __launch_bounds__(kTcThreads, 1) tc_forward_kernel_t(TcNet tc, TcArgs a, EnvFuse ef)
{
    TC_TRACE(0);
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *Ahi = smem, *Alo = smem + tc.a_bytes, *W = smem + 2 * tc.a_bytes;
    float *acc = reinterpret_cast<float *>(W + tc.img_bytes);        // accumulator tile [tc.max_rows][tc.acc_ld]
    __shared__ uint64_t wbar, wbar2;                         // weights of layer 0 | every other layer + the biases
    __shared__ const float *rows[kTcTile];
    __shared__ float s_rew[kTcTile], s_done[kTcTile];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = warp & 3, half = warp >> 2;
    // trainer blockIdx.y of a grouped learner: its weight image, rows [r0, r0 + n) of the inputs / outputs, its keys
    const int grp = blockIdx.y;
    const size_t r0 = (size_t)grp * (size_t)a.n;
    const unsigned char *img = a.img + (size_t)grp * (size_t)a.img_stride;
    // The first thread of the last warp initialises the two mbarriers and issues the weight copies while the other warps
    // already gather the first tile; the CTA-wide barrier in front of the first weight wait publishes the barriers.
    constexpr int kCtl = kTcThreads - 32;
    const bool early_w = (a.pdl & kPdlEarlyWeights) != 0;
    // The image travels in two pieces: layer 0's hi|lo block first (all the first MMA needs), the other layers and the biases
    // behind it on a second barrier that is first waited for in layer 0's epilogue -- when the image can only be requested
    // after the dependent-launch wait (act after the optimiser step) half of its latency is covered by the first layer.
    const uint32_t w_split = tc.n_layers > 1 ? (uint32_t)tc.L[1].hi_off : (uint32_t)tc.img_bytes;
    auto stage_image = [&]() {
        fence_proxy_async();
        bulk_g2s_chunked(W, img, w_split, &wbar);
        if (w_split < (uint32_t)tc.img_bytes) bulk_g2s_chunked(W + w_split, img + w_split, (uint32_t)tc.img_bytes - w_split, &wbar2);
    };
    if (tid == kCtl) {
        mbar_init(&wbar, 1); mbar_init(&wbar2, 1); fence_barrier_init();
        if (early_w) stage_image();
    }
    TC_TRACE(1);
    // PDL prologue (common.cuh): the weight image may be fetched before the wait when the predecessor does not write
    // it (TD passes after the env step); the first tile's rows may be gathered before the wait when the predecessor
    // does not write them (act after the optimiser kernel: observations were written two kernels back).
    bool waited = (a.pdl & kPdlEarlyRows) == 0;
    if (waited) {
        pdl_wait();
        pdl_trigger();
        if (tid == kCtl && !early_w) stage_image();
    }
    const float *bias_all = reinterpret_cast<const float *>(W + tc.bias_base);

    // act mode: row b of the tile is simply obs[base + b] -- no replay sampling (Philox), no pointer table, no barrier
    constexpr bool direct = ACT;
    uint32_t pkey[4] = {0u, 0u, 0u, 0u};
    const BatchSrc src = direct ? a.src : trainer_src(a.src, grp, a.n, tc.in_dim);
    if (!direct) Philox::gen(src.key, src.epoch, 0x5A17ull, pkey);
    bool wready = false, w2ready = false;

    // R = real rows per tile (32 / 64 / 128, at most tc.max_rows).  A warpgroup's m64 MMA runs when its rows hold real
    // samples; accumulator rows >= R are computed from whatever SMEM follows the R-row operand (still inside this CTA's allocation) and never stored.
    // Small batches use R = 32 so that 4096 samples spread over 128 CTAs instead of 32.
    const int R = a.rows_per_tile, lgR = 31 - __clz(R);
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int base = tile * R;
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
        TC_TRACE(27);
        // ---- A operand of layer 0: gathered rows -> TF32 hi/lo, canonical K-major layout (4 loads in flight per thread).
        //      Item i = (chunk j = i / R, row r = i % R): consecutive lanes take consecutive rows of the same 16-byte chunk, so
        //      a quarter-warp's 16-byte stores cover one whole core-matrix column = 128 contiguous bytes, and no division.
        {
            const int K0 = tc.L[0].K_pad, chunks = K0 / 4, total = R * chunks;
            const uint32_t sbo = mma_sbo(K0);
            for (int i0 = tid; i0 < total; i0 += 4 * kTcThreads) {
                float4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + u * kTcThreads;
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (i < total) {
                        const int r = i & (R - 1), j = i >> lgR;
                        const float *rp = direct ? ((base + r < a.n) ? a.obs + (r0 + base + r) * tc.in_dim : nullptr) : rows[r];
                        if (rp && 4 * j < tc.in_dim) v[u] = __ldg(reinterpret_cast<const float4 *>(rp) + j);
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + u * kTcThreads;
                    if (i < total) {
                        const int r = i & (R - 1), j = i >> lgR;
                        float4 h, l;
                        tf32_split(v[u].x, h.x, l.x); tf32_split(v[u].y, h.y, l.y); tf32_split(v[u].z, h.z, l.z); tf32_split(v[u].w, h.w, l.w);
                        const uint32_t off = mma_off(r, 4 * j, sbo);
                        *reinterpret_cast<float4 *>(Ahi + off) = h;
                        *reinterpret_cast<float4 *>(Alo + off) = l;
                    }
                }
            }
        }
        TC_TRACE(2);
        if (!waited) {
            pdl_wait();
            pdl_trigger();
            waited = true;
            if (tid == kCtl && !early_w) stage_image();
        }
        if (!wready) {                                           // first tile: the control thread's barriers become visible
            __syncthreads();
            mbar_wait(&wbar, 0);
            wready = true;
        }
        TC_TRACE(3);
        fence_proxy_async();
        __syncthreads();
        TC_TRACE(4);

        for (int l = 0; l < tc.n_layers; ++l) {
            const TcLayer T = tc.L[l];
            mma_3xtf32<kMmaFwd, FIXED>(acc, tc.acc_ld, Ahi, Alo, W + T.hi_off, W + T.lo_off, mma_sbo(T.K_pad), T.N_pad, T.K_pad / 8, R);
            TC_TRACE(5 + 3 * l);
            if (!w2ready) { if (w_split < (uint32_t)tc.img_bytes) mbar_wait(&wbar2, 0); w2ready = true; }   // biases + the next layers' weights
            TC_TRACE(6 + 3 * l);
            const float *bias = bias_all + T.bias_off;
            const int row = quad * 32 + lane;
            const bool live = quad * 32 < R;                       // this warp's rows are real rows
            if (l + 1 < tc.n_layers) {
                // hidden layer epilogue on every thread (EpiSlice): bias + ReLU, re-split, write the next A operand (K_next = N_pad)
                const uint32_t sbon = mma_sbo(T.N_pad);
                const EpiSlice e(R, kTcThreads);
                for (int c = e.c0; c < T.N_pad; c += e.step) {
                    const float4 v = e.ld(acc, tc.acc_ld, c);
                    float4 h, lo4;
                    const float x0 = fmaxf(v.x + bias[c + 0], 0.f), x1 = fmaxf(v.y + bias[c + 1], 0.f);
                    const float x2 = fmaxf(v.z + bias[c + 2], 0.f), x3 = fmaxf(v.w + bias[c + 3], 0.f);
                    tf32_split(x0, h.x, lo4.x); tf32_split(x1, h.y, lo4.y); tf32_split(x2, h.z, lo4.z); tf32_split(x3, h.w, lo4.w);
                    const uint32_t off = mma_off(e.row, c, sbon);
                    *reinterpret_cast<float4 *>(Ahi + off) = h;
                    *reinterpret_cast<float4 *>(Alo + off) = lo4;
                }
                fence_proxy_async();
                __syncthreads();
                TC_TRACE(7 + 3 * l);
            } else {
                // head epilogue: Q row of this sample, then the mode's output
                if (half == 0 && live) {
                    float q[32];
                    acc_ld32(acc, tc.acc_ld, row, 0, q);
                    const int nA = tc.n_actions;
#pragma unroll
                    for (int j = 0; j < 32; ++j) q[j] += bias[j];
                    if (DUELING) {                                 // Q = V + A - mean(A)  (BaseCNN.py:138)
                        float s = 0.f;
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < nA) s += q[j];
                        const float mean = s / (float)nA;
                        float V = 0.f;
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j == nA) V = q[j];
#pragma unroll
                        for (int j = 0; j < 32; ++j) q[j] = V + q[j] - mean;
                    }
                    int best = 0; float bv = q[0];
#pragma unroll
                    for (int j = 1; j < 32; ++j) if (j < nA && q[j] > bv) { bv = q[j]; best = j; }
                    const int b = base + row;                               // trainer-local row
                    const size_t ob = r0 + b;                               // its row in the [G][n] inputs / outputs
                    if (b < a.n) {
                        if (a.q_out) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) if (j < nA) a.q_out[ob * nA + j] = q[j];
                        }
                        if (ACT) {
                            float u; int ra;
                            if (a.u_tape) { u = a.u_tape[ob]; ra = a.rand_tape ? a.rand_tape[ob] : 0; }
                            else {
                                uint32_t rr[4];
                                Philox::gen(trainer_key(a.key, kActSalt, grp), a.call, (uint64_t)b, rr);
                                u = Philox::u01(rr[0]);
                                ra = (int)(((uint64_t)rr[1] * (uint64_t)nA) >> 32);
                            }
                            a.actions[ob] = (u > a.eps || !a.is_train) ? best : ra;     // DuelingDQN_Trainer.py:89-97
                        } else if (!ACT && a.mode == kTcArgmax) {
                            a.actions[ob] = best;                                       // DDQN_Trainer.py:94
                        } else {
                            float nq = bv;                                              // DQN_Trainer.py:109
                            if (a.mode == kTcTdGather) {                                // DDQN_Trainer.py:95
                                const int as = a.actions[ob];
                                nq = 0.f;
#pragma unroll
                                for (int j = 0; j < 32; ++j) if (j == as) nq = q[j];
                            }
                            a.y_out[ob] = s_rew[row] + (a.gamma * nq * (1.f - s_done[row]));  // :99 / :114 / :171
                        }
                    }
                }
                __syncthreads();
            }
        }
        if (FUSE_ENV) {
            // the tile's actions are in global memory (written by this CTA before the barrier above)
            __shared__ EnvSmem<32> env_sm;
            for (int sb = 0; sb < R; sb += 32)
                env_block<true, 32, kTcThreads, false, 8>(ef.d, env_sm, base + sb, tid, UAVRL_ACT_DISCRETE27, a.actions, ef.obs_next,
                                                       ef.reward, ef.done, nullptr, nullptr, nullptr);
            __syncthreads();
        }
    }
    TC_TRACE(20);
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

typedef void (*ForwardKernel)(TcNet, TcArgs, EnvFuse);
template <bool F, bool A, bool D>
static ForwardKernel pick_fwd_x(bool fixed) { return fixed ? tc_forward_kernel_t<F, A, D, true> : tc_forward_kernel_t<F, A, D, false>; }
template <bool F, bool A>
static ForwardKernel pick_fwd_d(bool dueling, bool fixed) { return dueling ? pick_fwd_x<F, A, true>(fixed) : pick_fwd_x<F, A, false>(fixed); }
// the fused act + env step variant exists for the act mode only
static ForwardKernel pick_forward_kernel(bool fuse_env, bool act, bool dueling, bool fixed)
{
    if (fuse_env) return pick_fwd_d<true, true>(dueling, fixed);
    return act ? pick_fwd_d<false, true>(dueling, fixed) : pick_fwd_d<false, false>(dueling, fixed);
}

int tc_forward_rows_per_tile(const TcNet &tc, int n)
{
    const int n_sm = num_sms();
    return (n >= 128 * n_sm && tc.max_rows == 128) ? 128 : (n >= 64 * n_sm) ? 64 : 32;
}

int launch_tc_forward(uavrl_learner *l, const TcArgs &a_in, cudaStream_t st, const EnvFuse *fuse)
{
    TcArgs a = a_in;
    a.img_stride = l->tc.train_img_bytes;
    const int n_sm = num_sms();
    a.rows_per_tile = tc_forward_rows_per_tile(l->tc, a.n);
    a.n_tiles = (a.n + a.rows_per_tile - 1) / a.rows_per_tile;
    const int grid = a.n_tiles < n_sm ? a.n_tiles : n_sm;
    static const bool trace_on = getenv("UAVRL_TC_TRACE") != nullptr;
    long long *tr = nullptr;
    if (trace_on) { UAVRL_CUDA(cudaMalloc((void **)&tr, 32 * sizeof(long long))); UAVRL_CUDA(cudaMemset(tr, 0, 32 * sizeof(long long))); a.trace = tr; }
    // PDL chain state (see common.cuh): what this kernel may touch before its griddepcontrol.wait
    const int prev = (l->pdl_chain && g_pdl.load()) ? l->pdl_prev : kPdlNone;
    a.pdl = 0;
    if (prev != kPdlNone) {
        a.pdl = kPdlOn;
        if (a.mode == kTcAct) {
            if (prev == kPdlAdam) a.pdl |= kPdlEarlyRows;          // obs frame written by the env step, weights by Adam
            else if (prev == kPdlEnv) a.pdl |= kPdlEarlyWeights;   // collection-only loop: weights untouched, obs just written
        } else if (prev == kPdlEnv || prev == kPdlTd) {
            a.pdl |= kPdlEarlyWeights;                             // neither the env step nor a TD pass writes weight images
        }
    }
    EnvFuse ef;
    memset(&ef, 0, sizeof(ef));
    if (fuse) {
        ef = *fuse;
        UAVRL_CUDA(launch_kernel(pick_forward_kernel(true, a.mode == kTcAct, l->tc.dueling != 0, tc_fixed_chains(l->tc, false)), dim3(grid), dim3(kTcThreads), tc_smem_bytes(l->tc), st, a.pdl != 0, l->tc, a, ef));
        l->pdl_prev = l->pdl_chain ? kPdlEnv : kPdlNone;
    } else {
        UAVRL_CUDA(launch_kernel(pick_forward_kernel(false, a.mode == kTcAct, l->tc.dueling != 0, tc_fixed_chains(l->tc, false)), dim3(grid, l->G), dim3(kTcThreads), tc_smem_bytes(l->tc), st, a.pdl != 0, l->tc, a, ef));
        l->pdl_prev = l->pdl_chain ? (a.mode == kTcAct ? kPdlAct : kPdlTd) : kPdlNone;
    }
    UAVRL_LAUNCHED();
    if (trace_on) {
        long long h[32];
        UAVRL_CUDA(cudaStreamSynchronize(st));
        UAVRL_CUDA(cudaMemcpy(h, tr, sizeof(h), cudaMemcpyDeviceToHost));
        cudaFree(tr);
        fprintf(stderr, "[tc_trace] mode=%d n=%d R=%d grid=%d cycles since start:", a.mode, a.n, a.rows_per_tile, grid);
        for (int i = 1; i < 32; ++i) if (h[i]) fprintf(stderr, " [%d]=%lld", i, h[i] - h[0]);
        fprintf(stderr, "\n");
    }
    return 0;
}

int tc_init(uavrl_learner *l)
{
    std::vector<int32_t> hi, lo, hi2, lo2;
    l->tc_ok = false; l->tc_train_ok = false;
    if (tc_build(l->cfg, l->net, l->tc, hi, lo, hi2, lo2) != 0) return 0;
    const bool fixed = tc_fixed_chains(l->tc, false);
    size_t fwd_static = 0;                                       // the kernels' static shared memory (row table, barriers)
    for (int ac = 0; ac < 2; ++ac)
        for (int du = 0; du < 2; ++du) {
            cudaFuncAttributes fa;
            UAVRL_CUDA(cudaFuncGetAttributes(&fa, pick_forward_kernel(false, ac != 0, du != 0, fixed)));
            if (fa.sharedSizeBytes > fwd_static) fwd_static = fa.sharedSizeBytes;
        }
    if (tc_smem_bytes(l->tc) + fwd_static > 227 * 1024) return 0;
    const size_t P = (size_t)l->net.P;
    const size_t img = (size_t)l->tc.train_img_bytes;
    const size_t img_all = (size_t)l->G * img;                  // [G] images of a grouped learner
    UAVRL_CUDA(cudaMalloc((void **)&l->tc_img_local, img_all));
    UAVRL_CUDA(cudaMalloc((void **)&l->tc_img_target, img_all));
    UAVRL_CUDA(cudaMemset(l->tc_img_local, 0, img_all));
    UAVRL_CUDA(cudaMemset(l->tc_img_target, 0, img_all));
    int32_t **maps[] = { &l->tc_hi_map, &l->tc_lo_map, &l->tc_hi2_map, &l->tc_lo2_map };
    std::vector<int32_t> *src[] = { &hi, &lo, &hi2, &lo2 };
    for (int i = 0; i < 4; ++i) {
        UAVRL_CUDA(cudaMalloc((void **)maps[i], P * 4));
        UAVRL_CUDA(cudaMemcpy(*maps[i], src[i]->data(), P * 4, cudaMemcpyHostToDevice));
    }
    UAVRL_CUDA(cudaMalloc((void **)&l->y_buf, (size_t)l->G * l->cfg.batch_size * 4));
    UAVRL_CUDA(cudaMalloc((void **)&l->astar_buf, (size_t)l->G * l->cfg.batch_size * 4));
    for (int ac = 0; ac < 2; ++ac)
        for (int du = 0; du < 2; ++du)
            UAVRL_CUDA(cudaFuncSetAttribute(pick_forward_kernel(false, ac != 0, du != 0, fixed), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)tc_smem_bytes(l->tc)));
    {   // the fused act+step variant carries the env scratch as static shared memory on top: it must still fit one CTA
        l->fuse_ok = true;
        for (int du = 0; du < 2; ++du) {
            cudaFuncAttributes fa;
            UAVRL_CUDA(cudaFuncGetAttributes(&fa, pick_forward_kernel(true, true, du != 0, fixed)));
            if (fa.sharedSizeBytes + tc_smem_bytes(l->tc) > (size_t)227 * 1024) l->fuse_ok = false;
        }
        if (l->fuse_ok)
            for (int du = 0; du < 2; ++du)
                UAVRL_CUDA(cudaFuncSetAttribute(pick_forward_kernel(true, true, du != 0, fixed), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)tc_smem_bytes(l->tc)));
    }
    l->y_cap = l->cfg.batch_size;
    l->tc_ok = true;
    return tc_train_init(l);
}

}  // namespace uavrl
