// sac_discrete.cu -- SAC with discrete actions on device, sm_90a: the IS_Continuous = 0 branch of the SAC learner (sac.cu).
//
// Replaces (include/uavrl.h, "SAC, discrete actions"):
//   SAC_Trainer.get_action      Trainer/SAC_Trainer.py:449-454 (Categorical(actor(s)).sample())
//   SAC_Trainer.update          Trainer/SAC_Trainer.py:380-430 (discrete branch), calc_target :133-141, soft_update :145-147
//   PolicyNet_SAC               BaseClass/BaseCNN.py:296-327   fc1 -> ReLU -> fc2 -> ReLU -> fc3 -> softmax over A
//   QValueNet_SAC               BaseClass/BaseCNN.py:329-343   fc1 -> ReLU -> fc2 -> ReLU -> fc3: A Q-values of s
// Four tile kernels on the fp32 SMEM-resident MLP blocks (mlp_tile.cuh), one CTA = 32 rows, templated on GR (grouped) as the
// continuous kernels are:
//   sacd_target_kernel   p' = actor(s'), both TARGET critics on s', y = r~ + gamma (sum p' min(Q1t, Q2t) + alpha H') (1 - d)
//   sacd_critic_kernel   both critics on s, the gathered squared error (Q_k(s)[a] - y)^2, backward -> gradient partials
//   sacd_actor_kernel    the UPDATED critics on s (forward only), actor forward and backward through the softmax
//   sacd_act_kernel      softmax + inverse-CDF categorical draw, or argmax p
// The update's Adam steps, alpha step and soft target update are the continuous learner's (reduce_adam_kernel,
// sac_finish_kernel); the two branches share no per-row math, so they share no tile kernel either.
#include "sac.cuh"
#include "mlp_tile.cuh"

namespace uavrl {

// Trainer g's share of a launch (gridDim.y = G; GR = false folds every offset to trainer 0)
template <bool GR> __device__ __forceinline__ int sacd_g() { return GR ? (int)blockIdx.y : 0; }
template <bool GR> __device__ __forceinline__ BatchSrc sacd_src(const SacdArgs &a) { return trainer_src(a.src, sacd_g<GR>(), a.B, a.actor.in_dim); }
template <bool GR> __device__ __forceinline__ uint64_t sacd_sample_key(const SacdArgs &a) { return trainer_key(a.src.key, kSampleSalt, sacd_g<GR>()); }
template <bool GR> __device__ __forceinline__ const float *sacd_img(const float *img, const NetDev &n) { return img + (size_t)sacd_g<GR>() * n.smem_w_floats; }
template <bool GR> __device__ __forceinline__ float *sacd_td(const SacdArgs &a) { return a.td + (size_t)sacd_g<GR>() * a.B; }
template <bool GR> __device__ __forceinline__ size_t sacd_part() { return (size_t)sacd_g<GR>() * gridDim.x + blockIdx.x; }

// softmax over row[0, A) in place: max-shifted, expf, summed left to right, divided (F.softmax, dim = 1)
__device__ __forceinline__ void softmax_row(float *row, int A)
{
    float m = row[0];
    for (int j = 1; j < A; ++j) m = fmaxf(m, row[j]);
    float s = 0.f;
    for (int j = 0; j < A; ++j) { const float e = expf(row[j] - m); row[j] = e; s += e; }
    for (int j = 0; j < A; ++j) row[j] = row[j] / s;
}

// backward of a whole network for the tile: dY (head gradient plane, [32][gld], zero in columns [A, 32)) -> parameter gradients
// into gpart; the forward's planes live at planes + n.act_off.  dY and dX ping-pong.
__device__ __forceinline__ void sacd_backward_tile(const NetDev &n, const float *sw, const float *planes, float *dY, float *dX, int gld, float *gpart,
                                   bool accumulate)
{
    for (int l = n.n_layers - 1; l >= 0; --l) {
        const LayerDev &L = n.L[l];
        const float *Xin = planes + n.act_off[l];
        const int ldx = n.act_ld[l];
        layer_backward_dw(dY, gld, Xin, ldx, gpart, L, accumulate);
        if (l > 0) {
            layer_backward_dx(dY, gld, sw + L.smem_w, Xin, ldx, dX, gld, L.in, L.out);
            // the next layer_backward_dx reads dX up to round_up(in, 4): the pad must be zero, not what the plane held
            const int pad = round_up(L.in, 4) - L.in;
            if (pad && threadIdx.x < kTile * pad) dX[(threadIdx.x / pad) * gld + L.in + threadIdx.x % pad] = 0.f;
            __syncthreads();
            float *tmp = dY; dY = dX; dX = tmp;
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------ TD target (calc_target, :133-141)
template <bool GR>
__global__ void __launch_bounds__(kNetThreads) sacd_target_kernel(SacdArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor, &cn = a.critic;
    float *RA = smem, *WT1 = RA + an.smem_total_floats, *WT2 = WT1 + cn.smem_w_floats;
    float *P = WT2 + cn.smem_w_floats, *q1 = P + kTile * 32, *q2 = q1 + kTile * 32;
    __shared__ uint64_t bar[3];
    __shared__ const float *rows[kTile];
    __shared__ float s_r[kTile], s_d[kTile];
    if (threadIdx.x == 0) { for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        stage_weights(an, sacd_img<GR>(a.img_actor, an), RA, &bar[0]); stage_weights(cn, sacd_img<GR>(a.img_t1, cn), WT1, &bar[1]);
        stage_weights(cn, sacd_img<GR>(a.img_t2, cn), WT2, &bar[2]);
    }
    uint32_t pkey[4];
    Philox::gen(sacd_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
    const float alpha = expf(a.log_alpha[3 * sacd_g<GR>()]);
    const int A = an.n_actions;
    float *X0 = RA + an.act_off[0];
    const int ld0 = an.act_ld[0];
    bool ready = false;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s2 = nullptr; tr.r = 0.f; tr.d = 0.f;
            if (gb < a.B) tr = resolve_transition(sacd_src<GR>(a), gb, an.in_dim, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s2 : nullptr; s_r[threadIdx.x] = tr.r; s_d[threadIdx.x] = tr.d;
        }
        __syncthreads();
        load_rows(rows, X0, ld0, an.in_dim);
        if (!ready) { for (int i = 0; i < 3; ++i) mbar_wait(&bar[i], 0); ready = true; }
        __syncthreads();
        // the three networks read the same input plane; each forward rewrites the trunk planes after it
        net_forward(an, RA, X0, ld0, RA, true, nullptr, nullptr, P);
        net_forward(cn, WT1, X0, ld0, RA, true, nullptr, nullptr, q1);
        net_forward(cn, WT2, X0, ld0, RA, true, nullptr, nullptr, q2);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            if (gb < a.B) {
                float *p = P + b * 32;
                softmax_row(p, A);
                float H = 0.f, m = 0.f;
                for (int j = 0; j < A; ++j) {
                    H -= p[j] * logf(p[j] + 1e-8f);
                    m += p[j] * fminf(q1[b * 32 + j], q2[b * 32 + j]);
                }
                const float r = (s_r[b] + 10.f) / 10.f;                               // reward shaping (:390)
                sacd_td<GR>(a)[gb] = r + a.gamma * (m + alpha * H) * (1.f - s_d[b]);
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ critic update (:397-406)
template <bool GR>
__global__ void __launch_bounds__(kNetThreads) sacd_critic_kernel(SacdArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &cn = a.critic;
    const int gld = a.gld;
    float *RC = smem, *WC2 = RC + cn.smem_total_floats;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * gld, *Q = dYb + kTile * gld;
    __shared__ uint64_t bar[2];
    __shared__ const float *rows[kTile];
    __shared__ int s_a[kTile];
    __shared__ float s_y[kTile], s_sq[kTile], s_acc[2];                // s_acc: thread 0's squared-error sums
    if (threadIdx.x == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) { stage_weights(cn, sacd_img<GR>(a.img_c1, cn), RC, &bar[0]); stage_weights(cn, sacd_img<GR>(a.img_c2, cn), WC2, &bar[1]); }
    // the sample key, the sums and the plane addresses are re-derived where they are used: nothing lives in registers across
    // the tile loop's layer calls
    if (threadIdx.x == 0) { s_acc[0] = 0.f; s_acc[1] = 0.f; }
    bool ready = false;
    int iter = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr; tr.a = 0;
            uint32_t pkey[4];
            Philox::gen(sacd_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
            if (gb < a.B) tr = resolve_transition(sacd_src<GR>(a), gb, cn.in_dim, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr; s_a[threadIdx.x] = tr.a;
            s_y[threadIdx.x] = (gb < a.B) ? sacd_td<GR>(a)[gb] : 0.f;
        }
        __syncthreads();
        load_rows(rows, RC + cn.act_off[0], cn.act_ld[0], cn.in_dim);
        if (!ready) { mbar_wait(&bar[0], 0); mbar_wait(&bar[1], 0); ready = true; }
        __syncthreads();
        for (int which = 0; which < 2; ++which) {
            const float *sw = which ? WC2 : RC;
            net_forward(cn, sw, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, Q);
            if (threadIdx.x < kTile) {
                const int b = threadIdx.x, gb = t * kTile + b;
                float *g = dYa + b * gld;
                for (int o = 0; o < 32; ++o) g[o] = 0.f;
                float e2 = 0.f;
                if (gb < a.B) {                                                     // Q_k(s).gather(1, a)
                    const float diff = Q[b * 32 + s_a[b]] - s_y[b];
                    e2 = diff * diff;
                    g[s_a[b]] = 2.f * diff * a.inv_b;
                }
                s_sq[b] = e2;
            }
            __syncthreads();
            if (threadIdx.x == 0) { float s = 0.f; for (int b = 0; b < kTile; ++b) s += s_sq[b]; s_acc[which] += s; }
            sacd_backward_tile(cn, sw, RC, dYa, dYb, gld, (which ? a.part_c2 : a.part_c1) + sacd_part<GR>() * cn.P, iter > 0);
        }
    }
    if (threadIdx.x == 0) { a.stat[sacd_part<GR>() * 4 + 0] = s_acc[0]; a.stat[sacd_part<GR>() * 4 + 1] = s_acc[1]; }
}

// ------------------------------------------------------------------ actor update (:408-419)
// L = mean(-alpha H - sum p min(Q1, Q2)) with H = -sum p log(p + 1e-8); Q does not depend on the actor, so per row
// dL/dp_j = (alpha (log(p_j + 1e-8) + p_j / (p_j + 1e-8)) - min_j) / B, then the softmax Jacobian dz_i = p_i (g_i - sum_j p_j g_j)
// Its three resident networks take one SM's shared memory, so one CTA per SM is what runs anyway: minBlocks = 1 lets the
// compiler keep the per-row epilogue in registers (no spills)
template <bool GR>
__global__ void __launch_bounds__(kNetThreads, 1) sacd_actor_kernel(SacdArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor, &cn = a.critic;
    const int gld = a.gld;
    float *RA = smem, *WC1 = RA + an.smem_total_floats, *WC2 = WC1 + cn.smem_w_floats;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * gld, *P = dYb + kTile * gld, *q1 = P + kTile * 32, *q2 = q1 + kTile * 32;
    __shared__ uint64_t bar[3];
    __shared__ const float *rows[kTile];
    __shared__ float s_l[kTile], s_e[kTile], s_acc[3];                 // s_acc: thread 0's loss and entropy sums, alpha
    if (threadIdx.x == 0) { for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        stage_weights(an, sacd_img<GR>(a.img_actor, an), RA, &bar[0]); stage_weights(cn, sacd_img<GR>(a.img_c1, cn), WC1, &bar[1]);
        stage_weights(cn, sacd_img<GR>(a.img_c2, cn), WC2, &bar[2]);
    }
    // as in the critic kernel, nothing but the loop counters lives in registers across the layer calls
    if (threadIdx.x == 0) { s_acc[0] = 0.f; s_acc[1] = 0.f; s_acc[2] = expf(a.log_alpha[3 * sacd_g<GR>()]); }
    int iter = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr;
            uint32_t pkey[4];
            Philox::gen(sacd_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
            if (gb < a.B) tr = resolve_transition(sacd_src<GR>(a), gb, an.in_dim, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr;
        }
        __syncthreads();
        load_rows(rows, RA + an.act_off[0], an.act_ld[0], an.in_dim);
        if (iter == 0) for (int i = 0; i < 3; ++i) mbar_wait(&bar[i], 0);
        __syncthreads();
        net_forward(cn, WC1, RA + an.act_off[0], an.act_ld[0], RA, true, nullptr, nullptr, q1);
        net_forward(cn, WC2, RA + an.act_off[0], an.act_ld[0], RA, true, nullptr, nullptr, q2);
        net_forward(an, RA, RA + an.act_off[0], an.act_ld[0], RA, true, nullptr, nullptr, P);   // the planes now hold the actor's trunk
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            float *g = dYa + b * gld;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            float l = 0.f, H = 0.f;
            if (gb < a.B) {
                const int A = an.n_actions;
                const float alpha = s_acc[2];
                float *p = P + b * 32;
                softmax_row(p, A);
                float m = 0.f, dot = 0.f;
                for (int j = 0; j < A; ++j) {
                    const float lp = logf(p[j] + 1e-8f), mn = fminf(q1[b * 32 + j], q2[b * 32 + j]);
                    H -= p[j] * lp;
                    m += p[j] * mn;
                    const float gj = (alpha * (lp + p[j] / (p[j] + 1e-8f)) - mn) * a.inv_b;
                    g[j] = gj;
                    dot += p[j] * gj;
                }
                for (int j = 0; j < A; ++j) g[j] = p[j] * (g[j] - dot);
                l = -alpha * H - m;
            }
            s_l[b] = l; s_e[b] = H;
        }
        __syncthreads();
        if (threadIdx.x == 0) { float s = 0.f, e = 0.f; for (int b = 0; b < kTile; ++b) { s += s_l[b]; e += s_e[b]; } s_acc[0] += s; s_acc[1] += e; }
        sacd_backward_tile(an, RA, RA, dYa, dYb, gld, a.part_a + sacd_part<GR>() * an.P, iter > 0);
    }
    if (threadIdx.x == 0) { a.stat[sacd_part<GR>() * 4 + 2] = s_acc[0]; a.stat[sacd_part<GR>() * 4 + 3] = s_acc[1]; }
}

// ------------------------------------------------------------------ get_action (:449-454)
// Trainer blockIdx.y acts for rows [g n, (g + 1) n).  One uniform u per row (the tape, or Philox(key of trainer g, ctr, row)
// word 0); the action is the smallest k with u sum(p) < p_0 + ... + p_k (fp32, left to right), else the last k with p_k > 0.
// MEAN: argmax p, the lowest index on ties; nothing is drawn.
template <bool GR, bool MEAN>
__global__ void __launch_bounds__(kNetThreads) sacd_act_kernel(SacdArgs a, const float *__restrict__ obs, int n, const float *__restrict__ u_tape,
                                                               int32_t *__restrict__ actions)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor;
    float *RA = smem, *P = RA + an.smem_total_floats;
    __shared__ uint64_t bar;
    __shared__ const float *rows[kTile];
    const int g = sacd_g<GR>();
    const int A = an.n_actions;
    const float *img = sacd_img<GR>(a.img_actor, an);
    obs += (size_t)g * n * an.in_dim; actions += (size_t)g * n;
    if (u_tape) u_tape += (size_t)g * n;
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) stage_weights(an, img, RA, &bar);
    bool ready = false;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        if (threadIdx.x < kTile) rows[threadIdx.x] = (t * kTile + threadIdx.x < n) ? obs + (size_t)(t * kTile + threadIdx.x) * an.in_dim : nullptr;
        __syncthreads();
        load_rows(rows, RA + an.act_off[0], an.act_ld[0], an.in_dim);
        if (!ready) { mbar_wait(&bar, 0); ready = true; }
        __syncthreads();
        net_forward(an, RA, RA + an.act_off[0], an.act_ld[0], RA, true, nullptr, nullptr, P);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            if (gb < n) {
                float *p = P + b * 32;
                softmax_row(p, A);
                int k;
                if (MEAN) {
                    k = argmax_row(p, A);
                } else {
                    float u;
                    if (u_tape) {
                        u = u_tape[gb];
                    } else {
                        uint32_t r[4];
                        Philox::gen(trainer_key(a.key, a.salt, g), a.ctr, (uint64_t)gb, r);
                        u = Philox::u01(r[0]);
                    }
                    float s = 0.f;
                    for (int j = 0; j < A; ++j) s += p[j];
                    const float x = u * s;
                    float c = 0.f;
                    k = -1;
                    for (int j = 0; j < A && k < 0; ++j) { c += p[j]; if (x < c) k = j; }
                    if (k < 0)
                        for (int j = A - 1; j >= 0 && k < 0; --j) if (p[j] > 0.f) k = j;
                    if (k < 0) k = A - 1;
                }
                actions[gb] = k;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ host side
size_t sacd_smem_dyn(const SacShape &s, int k)
{
    const size_t A = s.actor.smem_total_floats, C = s.critic.smem_total_floats, W = s.critic.smem_w_floats, H = kTile * 32,
                 D = (size_t)kTile * s.gld;
    switch (k) {
    case kSacdTarget: return (A + 2 * W + 3 * H) * 4;
    case kSacdCritic: return (C + W + 2 * D + H) * 4;
    case kSacdActor: return (A + 2 * W + 2 * D + 3 * H) * 4;
    default: return (A + H) * 4;
    }
}

int sacd_smem_total(const SacShape &s, size_t out[4])
{
    const void *k[4] = { (const void *)sacd_target_kernel<true>, (const void *)sacd_critic_kernel<true>, (const void *)sacd_actor_kernel<true>,
                         (const void *)sacd_act_kernel<true, false> };   // the one-trainer instances declare the same static smem
    for (int i = 0; i < 4; ++i) {
        cudaFuncAttributes fa;
        UAVRL_CUDA(cudaFuncGetAttributes(&fa, k[i]));
        out[i] = sacd_smem_dyn(s, i) + fa.sharedSizeBytes;
    }
    return 0;
}

int sacd_raise_smem(const SacShape &s)
{
    int rc;
    const size_t t = sacd_smem_dyn(s, kSacdTarget), c = sacd_smem_dyn(s, kSacdCritic), a = sacd_smem_dyn(s, kSacdActor),
                 x = sacd_smem_dyn(s, kSacdAct);
    if ((rc = raise_dyn_smem(sacd_target_kernel<false>, t)) || (rc = raise_dyn_smem(sacd_target_kernel<true>, t)) ||
        (rc = raise_dyn_smem(sacd_critic_kernel<false>, c)) || (rc = raise_dyn_smem(sacd_critic_kernel<true>, c)) ||
        (rc = raise_dyn_smem(sacd_actor_kernel<false>, a)) || (rc = raise_dyn_smem(sacd_actor_kernel<true>, a)) ||
        (rc = raise_dyn_smem(sacd_act_kernel<false, false>, x)) || (rc = raise_dyn_smem(sacd_act_kernel<true, false>, x)) ||
        (rc = raise_dyn_smem(sacd_act_kernel<false, true>, x)) || (rc = raise_dyn_smem(sacd_act_kernel<true, true>, x)))
        return rc;
    return 0;
}

int launch_sacd_phase(int k, const SacdArgs &a, int grid, int G, cudaStream_t st)
{
    const SacShape sh{ a.actor, a.critic, a.gld };
    const size_t sm = sacd_smem_dyn(sh, k);
    const dim3 tiles(grid, G);
    switch (k) {
    case kSacdTarget:
        if (G > 1) sacd_target_kernel<true><<<tiles, kNetThreads, sm, st>>>(a);
        else sacd_target_kernel<false><<<grid, kNetThreads, sm, st>>>(a);
        break;
    case kSacdCritic:
        if (G > 1) sacd_critic_kernel<true><<<tiles, kNetThreads, sm, st>>>(a);
        else sacd_critic_kernel<false><<<grid, kNetThreads, sm, st>>>(a);
        break;
    default:
        if (G > 1) sacd_actor_kernel<true><<<tiles, kNetThreads, sm, st>>>(a);
        else sacd_actor_kernel<false><<<grid, kNetThreads, sm, st>>>(a);
        break;
    }
    UAVRL_LAUNCHED();
    return 0;
}

int launch_sacd_act_kernel(const SacdArgs &a, const float *obs, int n, const float *u, bool mean, int32_t *actions, int grid, int G,
                           cudaStream_t st)
{
    const SacShape sh{ a.actor, a.critic, a.gld };
    const size_t sm = sacd_smem_dyn(sh, kSacdAct);
    const dim3 tiles(grid, G);
    if (mean && G > 1) sacd_act_kernel<true, true><<<tiles, kNetThreads, sm, st>>>(a, obs, n, nullptr, actions);
    else if (mean) sacd_act_kernel<false, true><<<grid, kNetThreads, sm, st>>>(a, obs, n, nullptr, actions);
    else if (G > 1) sacd_act_kernel<true, false><<<tiles, kNetThreads, sm, st>>>(a, obs, n, u, actions);
    else sacd_act_kernel<false, false><<<grid, kNetThreads, sm, st>>>(a, obs, n, u, actions);
    UAVRL_LAUNCHED();
    return 0;
}

}  // namespace uavrl
