// sac.cu -- SAC (continuous actions) learner on device, sm_90a: actor + twin critics + targets, learnable alpha.
//
// Replaces (SURVEY.md section 8a row a-14, BASELINE config 5):
//   SAC_Trainer.get_action      Trainer/SAC_Trainer.py:444-448
//   SAC_Trainer.update          Trainer/SAC_Trainer.py:325-379 (continuous branch), calc_target :122-131,
//                               soft_update :145-147
//   PolicyNetContinuous_SAC     BaseClass/BaseCNN.py:459-483   (mu = tanh, sigma = tanh(softplus), rsample, tanh squash,
//                               log-prob correction with tanh applied twice, :481)
//   QValueNetContinuous_SAC     BaseClass/BaseCNN.py:486-500   (input [s, a], output width = action_dim: the TD target and
//                               all losses are [B, action_dim]-shaped -- kept)
// Three tile kernels on the fp32 SMEM-resident MLP blocks (mlp_tile.cuh), one CTA = 32 sampled transitions:
//   sac_target_kernel   a', log pi(a'|s') from the actor, min of the two TARGET critics -> td[B][A]
//   sac_critic_kernel   both critics: forward on [s, a], MSE against td, backward -> gradient partials
//   sac_actor_kernel    actor forward on s (fresh noise), the UPDATED critics on [s, a_new], loss, backward through the
//                       critics to the action inputs, through tanh / softplus / the reparameterisation to the actor
// then reduce_adam_kernel per network and sac_finish_kernel (alpha step, soft target update).
// A grouped learner (uavrl_sac_create_trainers) holds G independent SAC trainers of one shape: every kernel takes the trainer
// from blockIdx.y (gridDim.y = G) and offsets its weight images, rows, noise key, log_alpha and scratch by it (sac_g and the
// helpers after it).
// sac_federate_kernel is Federated_Learning_AC (Envs/PathPlan_City.py:590-601) across those trainers' actors.
// A discrete learner (cfg.discrete, SAC_Trainer's IS_Continuous = 0 branch) shares this handle, its Adam, alpha and soft-update
// steps and its entry points; its four tile kernels live in sac_discrete.cu.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "sac.cuh"
#include "mlp_tile.cuh"

namespace uavrl {

constexpr int kSacA = 2;                 // action_dim of the reference's UAV task (config/Trainer.xml:8,21)
// row stride of the gradient ping-pong planes: a learner's sac_gld() = max(64, round_up(hidden, 32)), the columns
// layer_backward_dw reads.  The critic kernel also stages s rows across both planes at stride 2 gld (obs_dim <= 124 <= 2 x 64)
__host__ __device__ inline int sac_gld(int hidden) { const int w = round_up(hidden, 32); return w > 64 ? w : 64; }

struct SacHyper { float actor_lr, critic_lr, alpha_lr, target_entropy, gamma, tau, bound; };

// Every per-trainer array below is [G][...] (G = gridDim.y); the comments give one trainer's block.
struct SacArgs {
    NetDev actor, critic;
    BatchSrc src;
    int32_t B, n_tiles;                  // per trainer
    int32_t Bg;                          // rows the losses average over: B, or the global batch of a data-parallel update
    int32_t gld;                         // row stride of the gradient planes (sac_gld)
    const float *img_actor, *img_c1, *img_c2, *img_t1, *img_t2;   // [G][smem_w_floats] weight images
    const float *eps;                    // [B][A] injected noise (nullptr -> Philox Box-Muller)
    uint64_t key, ctr;                   // noise key of trainer 0 (trainer g: trainer_key(key, kNoiseSalt, g)), counter (shared)
    const float *log_alpha;              // [3]: log_alpha, its Adam exp_avg, exp_avg_sq
    float *td;                           // [B][A]
    float *part_a, *part_c1, *part_c2;   // gradient partials [grid][P]
    float *stat;                         // [grid][4]: critic-1 sq-err sum, critic-2 sq-err sum, actor-loss sum, entropy sum
    SacHyper h;
};

constexpr uint64_t kNoiseSalt = 0x5AC5ull;   // reparameterisation noise of a learner seeded `seed`: key seed ^ kNoiseSalt

// The tile kernels are templated on GR (grouped): a one-trainer learner launches GR = false, where the trainer index is the
// constant 0 and every offset below folds away, so it runs the code of a learner that knows nothing of trainers.
// Trainer g's share of the launch, evaluated where it is used (kept out of registers across the tile loop): its rows, weight
// images, noise key and stream, log_alpha, TD targets and partial slots.
template <bool GR> __device__ __forceinline__ int sac_g() { return GR ? (int)blockIdx.y : 0; }
template <bool GR> __device__ __forceinline__ BatchSrc sac_src(const SacArgs &a) { return trainer_src(a.src, sac_g<GR>(), a.B, a.actor.in_dim); }
template <bool GR> __device__ __forceinline__ uint64_t sac_sample_key(const SacArgs &a) { return trainer_key(a.src.key, kSampleSalt, sac_g<GR>()); }
template <bool GR> __device__ __forceinline__ const float *sac_img(const float *img, const NetDev &n) { return img + (size_t)sac_g<GR>() * n.smem_w_floats; }
template <bool GR> __device__ __forceinline__ const float *sac_eps(const SacArgs &a) { return a.eps ? a.eps + (size_t)sac_g<GR>() * a.B * kSacA : nullptr; }
template <bool GR> __device__ __forceinline__ uint64_t sac_noise_key(const SacArgs &a) { return trainer_key(a.key, kNoiseSalt, sac_g<GR>()); }   // (seed + g) ^ salt
template <bool GR> __device__ __forceinline__ float *sac_td(const SacArgs &a) { return a.td + (size_t)sac_g<GR>() * a.B * kSacA; }
template <bool GR> __device__ __forceinline__ size_t sac_part() { return (size_t)sac_g<GR>() * gridDim.x + blockIdx.x; }

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ void noise2(const float *eps, uint64_t key, uint64_t ctr, int gb, float &e0, float &e1)
{
    if (eps) { e0 = eps[2 * gb]; e1 = eps[2 * gb + 1]; return; }
    uint32_t r[4];
    Philox::gen(key, ctr, (uint64_t)gb, r);
    const float u0 = ((float)(r[0] >> 8) + 0.5f) * (1.0f / 16777216.0f), u1 = Philox::u01(r[1]);
    const float rad = sqrtf(-2.f * logf(u0));
    e0 = rad * cospif(2.f * u1); e1 = rad * sinpif(2.f * u1);
}

// per-sample quantities of PolicyNetContinuous_SAC.forward (BaseCNN.py:471-483) from the head pre-activations
struct ActorOut { float mu, sd, ps, a, t, logp; };
__device__ __forceinline__ ActorOut actor_point(float pm, float ps, float eps)
{
    ActorOut o;
    o.ps = ps;
    o.mu = tanhf(pm);
    o.sd = tanhf(softplus_f(ps));
    const float xs = o.mu + o.sd * eps;                                             // rsample
    const float var = o.sd * o.sd, dev = xs - o.mu;
    const float lp = -(dev * dev) / (2.f * var) - logf(o.sd) - 0.91893853320467274178f;   // Normal.log_prob
    o.a = tanhf(xs);
    o.t = tanhf(o.a);                                                               // tanh applied twice (:481)
    o.logp = lp - logf(1.f - o.t * o.t + 1e-7f);
    return o;
}

// actor on the tile in plane X (ld): trunk output -> actor plane 1, head pre-activations -> head[32][32]
__device__ void actor_forward_tile(const NetDev &an, const float *ra, float *head)
{
    const LayerDev &L0 = an.L[0], &L1 = an.L[1];
    layer_forward(ra + an.act_off[0], an.act_ld[0], ra + L0.smem_w, ra + L0.smem_b, const_cast<float *>(ra) + an.act_off[1], an.act_ld[1], L0.in, L0.out, true);
    __syncthreads();
    layer_forward(ra + an.act_off[1], an.act_ld[1], ra + L1.smem_w, ra + L1.smem_b, head, 32, L1.in, L1.out, false);
    __syncthreads();
}

// critic input plane = [s (copied from the actor's input plane or loaded rows), a, 0-pad]
__device__ void build_critic_input(const float *S, int lds, int obs_dim, float *XC, int ldc, const float (*act)[kSacA])
{
    for (int i = threadIdx.x; i < kTile * obs_dim; i += blockDim.x) {
        const int b = i / obs_dim, k = i - b * obs_dim;
        XC[b * ldc + k] = S[b * lds + k];
    }
    if (threadIdx.x < kTile) {
        const int b = threadIdx.x;
        for (int j = 0; j < kSacA; ++j) XC[b * ldc + obs_dim + j] = act[b][j];
        for (int k = obs_dim + kSacA; k < round_up(obs_dim + kSacA, 4); ++k) XC[b * ldc + k] = 0.f;
    }
}

// backward of one critic for the tile: dY (head gradient plane, [32][gld], zero beyond the 2 outputs) -> optional parameter
// gradients into gpart, optional action-input gradient dA[32][A].  Planes of the critic live at rc + act_off.
__device__ void critic_backward_tile(const NetDev &cn, const float *sw, const float *rc, float *dY, float *dX, int gld, float *gpart,
                                     bool accumulate, float (*dA)[kSacA], int obs_dim)
{
    for (int l = cn.n_layers - 1; l >= 0; --l) {
        const LayerDev &L = cn.L[l];
        const float *Xin = rc + cn.act_off[l];
        const int ldx = cn.act_ld[l];
        if (gpart) layer_backward_dw(dY, gld, Xin, ldx, gpart, L, accumulate);
        if (l > 0) {
            layer_backward_dx(dY, gld, sw + L.smem_w, Xin, ldx, dX, gld, L.in, L.out);
            // the next layer_backward_dx reads dX up to round_up(in, 4) and multiplies the pad by zero weights: the pad must be
            // zero, not whatever the plane held (0 x NaN is NaN)
            const int pad = round_up(L.in, 4) - L.in;
            if (pad && threadIdx.x < kTile * pad) dX[(threadIdx.x / pad) * gld + L.in + threadIdx.x % pad] = 0.f;
            __syncthreads();
            float *tmp = dY; dY = dX; dX = tmp;
        } else if (dA) {
            __syncthreads();
            // gradient w.r.t. the action inputs only: dA[b][j] = sum_o dZ1[b][o] * W1[o][obs+j]  (Wt row obs+j is contiguous in o)
            if (threadIdx.x < kTile * kSacA) {
                const int b = threadIdx.x / kSacA, j = threadIdx.x - b * kSacA;
                const int ldw = ldw_of(L.out);
                const float *w = sw + L.smem_w + (obs_dim + j) * ldw;
                float s = 0.f;
                for (int o = 0; o < L.out; ++o) s += dY[b * gld + o] * w[o];
                dA[b][j] = s;
            }
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------ TD target (calc_target, :122-131)
template <bool GR>
__global__ void __launch_bounds__(kNetThreads) sac_target_kernel(SacArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor, &cn = a.critic;
    float *RA = smem, *RT1 = RA + an.smem_total_floats, *WT2 = RT1 + cn.smem_total_floats;
    float *head = WT2 + cn.smem_w_floats, *q1 = head + kTile * 32, *q2 = q1 + kTile * 32;
    __shared__ uint64_t bar[3];
    __shared__ const float *rows[kTile];
    __shared__ float s_r[kTile], s_d[kTile], s_logp[kTile][kSacA], s_act[kTile][kSacA];
    if (threadIdx.x == 0) { for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        stage_weights(an, sac_img<GR>(a.img_actor, an), RA, &bar[0]); stage_weights(cn, sac_img<GR>(a.img_t1, cn), RT1, &bar[1]);
        stage_weights(cn, sac_img<GR>(a.img_t2, cn), WT2, &bar[2]);
    }
    uint32_t pkey[4];
    Philox::gen(sac_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
    const float alpha = expf(a.log_alpha[3 * sac_g<GR>()]);
    bool ready = false;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s2 = nullptr; tr.r = 0.f; tr.d = 0.f;
            if (gb < a.B) tr = resolve_transition(sac_src<GR>(a), gb, an.in_dim, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s2 : nullptr; s_r[threadIdx.x] = tr.r; s_d[threadIdx.x] = tr.d;
        }
        __syncthreads();
        load_rows(rows, RA + an.act_off[0], an.act_ld[0], an.in_dim);
        if (!ready) { for (int i = 0; i < 3; ++i) mbar_wait(&bar[i], 0); ready = true; }
        __syncthreads();
        actor_forward_tile(an, RA, head);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            float e[2] = { 0.f, 0.f };
            if (gb < a.B) noise2(sac_eps<GR>(a), sac_noise_key<GR>(a), a.ctr, gb, e[0], e[1]);
            for (int j = 0; j < kSacA; ++j) {
                const ActorOut o = actor_point(head[b * 32 + j], head[b * 32 + kSacA + j], e[j]);
                s_act[b][j] = o.a * a.h.bound; s_logp[b][j] = o.logp;
            }
        }
        __syncthreads();
        build_critic_input(RA + an.act_off[0], an.act_ld[0], an.in_dim, RT1 + cn.act_off[0], cn.act_ld[0], s_act);
        __syncthreads();
        net_forward(cn, RT1, RT1 + cn.act_off[0], cn.act_ld[0], RT1, true, nullptr, nullptr, q1);
        net_forward(cn, WT2, RT1 + cn.act_off[0], cn.act_ld[0], RT1, true, nullptr, nullptr, q2);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            if (gb < a.B)
                for (int j = 0; j < kSacA; ++j) {
                    const float nv = fminf(q1[b * 32 + j], q2[b * 32 + j]) + alpha * (-s_logp[b][j]);
                    sac_td<GR>(a)[(size_t)gb * kSacA + j] = s_r[b] + a.h.gamma * nv * (1.f - s_d[b]);
                }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ critic update (:343-360)
// PW (prioritised replay): row b's squared errors and head gradient are scaled by its importance weight w_b (src.is_w), so
// L_k = mean over B x A of w_b (Q_k - y)^2, and after critic 2 the row's priority error
// e_b = 0.5 (|min(Q1, Q2)_0 - y_0| + |min(Q1, Q2)_1 - y_1|) goes to src.abs_err (when given), from the critics before this step
template <bool GR, bool PW>
__global__ void __launch_bounds__(kNetThreads) sac_critic_kernel(SacArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &cn = a.critic;
    float *RC = smem, *WC2 = RC + cn.smem_total_floats;
    const int gld = a.gld;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * gld, *Q = dYb + kTile * gld;
    __shared__ uint64_t bar[2];
    __shared__ const float *rows[kTile];
    __shared__ float s_act[kTile][kSacA], s_sq[kTile];
    // PW: row weights; critic 1's outputs through critic 2; thread 0's squared-error sums and 1 / (Bg A) (kept out of registers)
    __shared__ float s_w[PW ? kTile : 1], s_q1[PW ? kTile : 1][kSacA], s_acc[3];
    if (threadIdx.x == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) { stage_weights(cn, sac_img<GR>(a.img_c1, cn), RC, &bar[0]); stage_weights(cn, sac_img<GR>(a.img_c2, cn), WC2, &bar[1]); }
    uint32_t pkey[4];                                                       // PW: derived per tile (kept out of registers)
    if constexpr (!PW) Philox::gen(sac_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
    const float inv = 1.f / ((float)a.Bg * (float)kSacA);
    float sq[2] = { 0.f, 0.f };
    if constexpr (PW) { if (threadIdx.x == 0) { s_acc[0] = s_acc[1] = 0.f; s_acc[2] = inv; } }
    bool ready = false;
    int iter = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr; tr.ax = tr.ay = 0.f;
            if constexpr (PW) Philox::gen(sac_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
            if (gb < a.B) tr = resolve_transition(sac_src<GR>(a), gb, cn.in_dim - kSacA, pkey);
            if constexpr (PW) s_w[threadIdx.x] = (gb < a.B) ? sac_src<GR>(a).is_w[gb] : 0.f;
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr; s_act[threadIdx.x][0] = tr.ax; s_act[threadIdx.x][1] = tr.ay;
        }
        __syncthreads();
        load_rows(rows, dYa, gld * 2, cn.in_dim - kSacA);                   // stage s in the (still unused) gradient planes: 32 x 2 gld
        __syncthreads();
        build_critic_input(dYa, gld * 2, cn.in_dim - kSacA, RC + cn.act_off[0], cn.act_ld[0], s_act);
        if (PW ? iter == 0 : !ready) { mbar_wait(&bar[0], 0); mbar_wait(&bar[1], 0); ready = true; }
        __syncthreads();
        for (int which = 0; which < 2; ++which) {
            const float *sw = which ? WC2 : RC;
            net_forward(cn, sw, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, Q);
            if (threadIdx.x < kTile) {
                const int b = threadIdx.x, gb = t * kTile + b;
                float *g = dYa + b * gld;
                for (int o = 0; o < 32; ++o) g[o] = 0.f;
                float e2 = 0.f;
                if (gb < a.B)
                    for (int j = 0; j < kSacA; ++j) {
                        const float diff = Q[b * 32 + j] - sac_td<GR>(a)[(size_t)gb * kSacA + j];
                        e2 += diff * diff;
                        if constexpr (PW) g[j] = 2.f * s_w[b] * diff * s_acc[2];
                        else g[j] = 2.f * diff * inv;
                    }
                if constexpr (PW) {
                    s_sq[b] = s_w[b] * e2;
                    if (which == 0) { s_q1[b][0] = Q[b * 32]; s_q1[b][1] = Q[b * 32 + 1]; }
                } else {
                    s_sq[b] = e2;
                }
            }
            __syncthreads();
            if (threadIdx.x == 0) { float s = 0.f; for (int b = 0; b < kTile; ++b) s += s_sq[b]; if constexpr (PW) s_acc[which] += s; else sq[which] += s; }
            critic_backward_tile(cn, sw, RC, dYa, dYb, gld, (which ? a.part_c2 : a.part_c1) + sac_part<GR>() * cn.P, iter > 0, nullptr, 0);
        }
        if constexpr (PW) {                                                 // Q still holds critic 2's outputs
            const int b = threadIdx.x, gb = t * kTile + b;
            float *abs_err = sac_src<GR>(a).abs_err;
            if (b < kTile && gb < a.B && abs_err) {
                const float *y = sac_td<GR>(a) + (size_t)gb * kSacA;
                const float m0 = fminf(s_q1[b][0], Q[b * 32]), m1 = fminf(s_q1[b][1], Q[b * 32 + 1]);
                abs_err[gb] = 0.5f * (fabsf(m0 - y[0]) + fabsf(m1 - y[1]));
            }
        }
    }
    if constexpr (PW) { if (threadIdx.x == 0) { sq[0] = s_acc[0]; sq[1] = s_acc[1]; } }
    if (threadIdx.x == 0) { a.stat[sac_part<GR>() * 4 + 0] = sq[0]; a.stat[sac_part<GR>() * 4 + 1] = sq[1]; }
}

// ------------------------------------------------------------------ actor update (:362-376)
template <bool GR>
__global__ void __launch_bounds__(kNetThreads) sac_actor_kernel(SacArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor, &cn = a.critic;
    float *RA = smem, *RC = RA + an.smem_total_floats, *WC2 = RC + cn.smem_total_floats;
    const int gld = a.gld;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * gld, *head = dYb + kTile * gld, *q1 = head + kTile * 32, *q2 = q1 + kTile * 32;
    __shared__ uint64_t bar[3];
    __shared__ const float *rows[kTile];
    __shared__ ActorOut s_o[kTile][kSacA];
    __shared__ float s_eps[kTile][kSacA], s_act[kTile][kSacA], s_dq1[kTile][kSacA], s_dq2[kTile][kSacA], s_dA1[kTile][kSacA],
        s_dA2[kTile][kSacA], s_l[kTile], s_e[kTile];
    if (threadIdx.x == 0) { for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        stage_weights(an, sac_img<GR>(a.img_actor, an), RA, &bar[0]); stage_weights(cn, sac_img<GR>(a.img_c1, cn), RC, &bar[1]);
        stage_weights(cn, sac_img<GR>(a.img_c2, cn), WC2, &bar[2]);
    }
    uint32_t pkey[4];
    Philox::gen(sac_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
    const float alpha = expf(a.log_alpha[3 * sac_g<GR>()]);
    const float inv = 1.f / ((float)a.Bg * (float)kSacA);
    float loss_acc = 0.f, ent_acc = 0.f;
    bool ready = false;
    int iter = 0;
    float *gpart = a.part_a + sac_part<GR>() * an.P;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr;
            if (gb < a.B) tr = resolve_transition(sac_src<GR>(a), gb, an.in_dim, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr;
        }
        __syncthreads();
        load_rows(rows, RA + an.act_off[0], an.act_ld[0], an.in_dim);
        if (!ready) { for (int i = 0; i < 3; ++i) mbar_wait(&bar[i], 0); ready = true; }
        __syncthreads();
        actor_forward_tile(an, RA, head);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            float e[2] = { 0.f, 0.f };
            if (gb < a.B) noise2(sac_eps<GR>(a), sac_noise_key<GR>(a), a.ctr, gb, e[0], e[1]);
            for (int j = 0; j < kSacA; ++j) {
                s_eps[b][j] = e[j];
                s_o[b][j] = actor_point(head[b * 32 + j], head[b * 32 + kSacA + j], e[j]);
                s_act[b][j] = s_o[b][j].a * a.h.bound;
            }
        }
        __syncthreads();
        build_critic_input(RA + an.act_off[0], an.act_ld[0], an.in_dim, RC + cn.act_off[0], cn.act_ld[0], s_act);
        __syncthreads();
        net_forward(cn, RC, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, q1);
        net_forward(cn, WC2, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, q2);     // planes now hold critic 2
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            float l = 0.f, en = 0.f;
            float *g = dYa + b * gld;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            for (int j = 0; j < kSacA; ++j) {
                const float v1 = q1[b * 32 + j], v2 = q2[b * 32 + j];
                const float gmin = (gb < a.B) ? -inv : 0.f;                                        // d loss / d min(q1, q2)
                s_dq1[b][j] = v1 < v2 ? gmin : (v1 > v2 ? 0.f : 0.5f * gmin);
                s_dq2[b][j] = v2 < v1 ? gmin : (v2 > v1 ? 0.f : 0.5f * gmin);
                g[j] = s_dq2[b][j];
                if (gb < a.B) { l += alpha * s_o[b][j].logp - fminf(v1, v2); en += -s_o[b][j].logp; }
            }
            s_l[b] = l; s_e[b] = en;
        }
        __syncthreads();
        if (threadIdx.x == 0) { float s = 0.f, e = 0.f; for (int b = 0; b < kTile; ++b) { s += s_l[b]; e += s_e[b]; } loss_acc += s; ent_acc += e; }
        critic_backward_tile(cn, WC2, RC, dYa, dYb, gld, nullptr, false, s_dA2, an.in_dim);              // d/d a through critic 2
        net_forward(cn, RC, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, q1);      // planes back to critic 1
        if (threadIdx.x < kTile) {
            float *g = dYa + threadIdx.x * gld;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            for (int j = 0; j < kSacA; ++j) g[j] = s_dq1[threadIdx.x][j];
        }
        __syncthreads();
        critic_backward_tile(cn, RC, RC, dYa, dYb, gld, nullptr, false, s_dA1, an.in_dim);               // d/d a through critic 1
        // through tanh squash, reparameterisation, tanh / softplus heads to the head pre-activations
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x;
            float *g = dYa + b * gld;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            const bool valid = (t * kTile + b) < a.B;
            for (int j = 0; j < kSacA; ++j) {
                const ActorOut o = s_o[b][j];
                const float glogp = valid ? alpha * inv : 0.f;
                const float dc_da = 2.f * o.t * (1.f - o.t * o.t) / (1.f - o.t * o.t + 1e-7f);
                const float dxs = (s_dA1[b][j] + s_dA2[b][j]) * a.h.bound * (1.f - o.a * o.a) + glogp * dc_da * (1.f - o.a * o.a);
                const float dsd = dxs * s_eps[b][j] + glogp * (-1.f / o.sd);
                g[j] = dxs * (1.f - o.mu * o.mu);                                                   // d / d (mu pre-activation)
                g[kSacA + j] = dsd * (1.f - o.sd * o.sd) * (o.ps > 20.f ? 1.f : sigmoid_f(o.ps));   // d / d (sigma pre-activation)
            }
        }
        __syncthreads();
        // actor backward: head (dW, dX), trunk (dW)
        {
            const LayerDev &L1 = an.L[1], &L0 = an.L[0];
            layer_backward_dw(dYa, gld, RA + an.act_off[1], an.act_ld[1], gpart, L1, iter > 0);
            layer_backward_dx(dYa, gld, RA + L1.smem_w, RA + an.act_off[1], an.act_ld[1], dYb, gld, L1.in, L1.out);
            __syncthreads();
            layer_backward_dw(dYb, gld, RA + an.act_off[0], an.act_ld[0], gpart, L0, iter > 0);
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) { a.stat[sac_part<GR>() * 4 + 2] = loss_acc; a.stat[sac_part<GR>() * 4 + 3] = ent_acc; }
}

// ------------------------------------------------------------------ alpha step + soft target update + scalar outputs
struct SacFinishArgs {
    int Pc, nparts;
    int img_floats;                      // per-trainer stride of the critic weight images
    float tau, alpha_lr, target_entropy, inv_n, step_size_scale, bc2_sqrt;
    int do_alpha;
};

// blockIdx.y = trainer g: its stat [nparts][4], scal [3], critics and targets [Pc], target images and out [4].  sums_c / sums_a
// (data-parallel, one trainer): the squared-error sums / the actor-loss and entropy sums over every rank, which then replace
// the stat partials
__global__ void sac_finish_kernel(SacFinishArgs f, const float *__restrict__ stat, const float *__restrict__ sums_c,
                                  const float *__restrict__ sums_a, float *__restrict__ scal, const float *__restrict__ c1,
                                  const float *__restrict__ c2, float *__restrict__ t1, float *__restrict__ t2, float *__restrict__ img_t1,
                                  float *__restrict__ img_t2, const int32_t *__restrict__ cmap, float *__restrict__ out)
{
    {
        const size_t g = blockIdx.y, gp = g * (size_t)f.Pc, gi = g * (size_t)f.img_floats;
        stat += g * 4 * (size_t)f.nparts; scal += 3 * g;
        c1 += gp; c2 += gp; t1 += gp; t2 += gp; img_t1 += gi; img_t2 += gi;
        if (out) out += 4 * g;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < f.Pc) {                                                           // soft_update (:145-147) with the updated critics
        const int im = cmap[i];
        const float a1 = t1[i] * (1.0f - f.tau) + c1[i] * f.tau, a2 = t2[i] * (1.0f - f.tau) + c2[i] * f.tau;
        t1[i] = a1; t2[i] = a2; img_t1[im] = a1; img_t2[im] = a2;
    }
    if (blockIdx.x == 0 && threadIdx.x < 32) {
        // the per-CTA loss / entropy partials: lane-strided sums, then a butterfly (one thread walking all of them serially is a
        // chain of dependent global loads).  A data-parallel exchange sums each rank's partials in this order, so one rank
        // reads 0 + its own sums
        float s0, s1, s2, s3;
        if (sums_c) {
            s0 = sums_c[0]; s1 = sums_c[1]; s2 = sums_a[0]; s3 = sums_a[1];
        } else {
            s0 = warp_column_sum(stat, f.nparts, 4, 0); s1 = warp_column_sum(stat, f.nparts, 4, 1);
            s2 = warp_column_sum(stat, f.nparts, 4, 2); s3 = warp_column_sum(stat, f.nparts, 4, 3);
        }
        if (threadIdx.x != 0) return;
        // alpha_loss = mean((entropy - target_entropy).detach() * exp(log_alpha))  (:372-376), Adam on log_alpha
        const float alpha = expf(scal[0]);
        const float g = (s3 * f.inv_n - f.target_entropy) * alpha;
        if (f.do_alpha) {
            float m = scal[1], v = scal[2];
            m = m + (g - m) * 0.1f;
            v = v * 0.999f + 0.001f * g * g;
            scal[0] = scal[0] - f.step_size_scale * (m / (sqrtf(v) / f.bc2_sqrt + 1e-8f));
            scal[1] = m; scal[2] = v;
        }
        if (out) { out[0] = s2 * f.inv_n; out[1] = s0 * f.inv_n; out[2] = s1 * f.inv_n; out[3] = g; }   // actor, critic1, critic2, alpha loss
    }
}

// the split data-parallel form's scalar words: columns j0 and j0 + 1 of the [nparts][4] stat partials, summed as the fused
// exchange and sac_finish_kernel sum them
__global__ void sac_stat_sums_kernel(const float *__restrict__ stat, int nparts, int j0, float *__restrict__ out)
{
    const float a = warp_column_sum(stat, nparts, 4, j0), b = warp_column_sum(stat, nparts, 4, j0 + 1);
    if (threadIdx.x == 0) { out[0] = a; out[1] = b; }
}

// get_action (:444-448): action = actor(state)[0] with fresh noise.  Trainer blockIdx.y acts for rows [g n, (g + 1) n).
// MEAN: the policy's mean action instead, tanh(mu) bound -- PolicyNetContinuous_SAC.forward with zero noise (the evaluation's
// deterministic policy, uavrl_sac_eval_run / uavrl_sac_act_mean); no noise is drawn.
template <bool GR, bool MEAN = false>
__global__ void __launch_bounds__(kNetThreads) sac_act_kernel(SacArgs a, const float *__restrict__ obs, int n, float *__restrict__ actions)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor;
    float *RA = smem, *head = RA + an.smem_total_floats;
    __shared__ uint64_t bar;
    __shared__ const float *rows[kTile];
    const int g = sac_g<GR>();
    const float *img = sac_img<GR>(a.img_actor, an), *eps = a.eps ? a.eps + (size_t)g * n * kSacA : nullptr;
    const uint64_t key = sac_noise_key<GR>(a);
    obs += (size_t)g * n * an.in_dim; actions += (size_t)g * n * kSacA;
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
        actor_forward_tile(an, RA, head);
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x, gb = t * kTile + b;
            if (MEAN && gb < n) {
                for (int j = 0; j < kSacA; ++j) actions[(size_t)gb * kSacA + j] = tanhf(tanhf(head[b * 32 + j])) * a.h.bound;
            } else if (gb < n) {
                float e[2];
                noise2(eps, key, a.ctr, gb, e[0], e[1]);
                for (int j = 0; j < kSacA; ++j) actions[(size_t)gb * kSacA + j] = actor_point(head[b * 32 + j], head[b * 32 + kSacA + j], e[j]).a * a.h.bound;
            }
        }
        __syncthreads();
    }
}

// Federated_Learning_AC (Envs/PathPlan_City.py:590-601): global = deepcopy(actor_0); global[k] += actor_i[k] for i = 1 .. G-1;
// every actor <- global.  The reference's division assigns into a temporary state_dict and is lost, so every actor becomes the
// float32 sum theta_0 + theta_1 + ... + theta_{G-1}, added left to right in trainer order.  One thread per actor parameter: the
// sum of the G actors [G][P] in `actors` goes to the n_out actors [n_out][P] in `out` (the same G actors, or a shard's own).
__global__ void sac_federate_kernel(int P, int G, const float *actors, int n_out, float *out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float s = actors[i];
    for (int g = 1; g < G; ++g) s = __fadd_rn(s, actors[(size_t)g * P + i]);
    for (int g = 0; g < n_out; ++g) out[(size_t)g * P + i] = s;
}

}  // namespace uavrl

using namespace uavrl;

// ------------------------------------------------------------------ host handle (sac.cuh)
// refuses a configuration before anything is allocated
static int sac_shape(const uavrl_sac_config &c, SacShape &sh)
{
    if (c.discrete != 0 && c.discrete != 1) return fail(UAVRL_ERR_INVALID, "discrete must be 0 (continuous actions) or 1 (discrete actions)");
    if (c.discrete) {                                          // PolicyNet_SAC / QValueNet_SAC: obs -> hidden -> hidden -> A
        if (c.act_dim < 2 || c.act_dim > 31) return fail(UAVRL_ERR_INVALID, "a discrete SAC learner's act_dim must be in [2, 31]");
        if (c.obs_dim <= 0 || c.obs_dim % 4 != 0 || c.obs_dim > kMaxDim)
            return fail(UAVRL_ERR_INVALID, "a discrete SAC learner's obs_dim must be a multiple of 4 in [4, 128]");
        if (c.hidden < 1 || c.hidden > kMaxDim) return fail(UAVRL_ERR_INVALID, "hidden must be in [1, 128]");
        int rc;
        const int32_t hh[2] = { c.hidden, c.hidden };
        if ((rc = build_mlp(c.obs_dim, 2, hh, c.act_dim, 0, sh.actor)) || (rc = build_mlp(c.obs_dim, 2, hh, c.act_dim, 0, sh.critic))) return rc;
        sh.gld = sac_gld(c.hidden);
        return 0;
    }
    if (c.act_dim != kSacA) return fail(UAVRL_ERR_INVALID, "act_dim must be 2 (the reference's UAV task)");
    if (c.obs_dim <= 0 || c.obs_dim % 4 != 0) return fail(UAVRL_ERR_INVALID, "obs_dim must be a multiple of 4");
    if (c.obs_dim > kMaxDim - kSacA) return fail(UAVRL_ERR_INVALID, "obs_dim must be at most 124 (the critic input obs_dim + 2 is at most 128)");
    if (c.hidden < 1 || c.hidden > kMaxDim) return fail(UAVRL_ERR_INVALID, "hidden must be in [1, 128]");
    int rc;
    const int32_t ha[1] = { c.hidden }, hc[2] = { c.hidden, c.hidden };
    if ((rc = build_mlp(c.obs_dim, 1, ha, kSacA, kSacA, sh.actor))) return rc;              // fc1 -> {fc_mu ; fc_std}
    if ((rc = build_mlp(c.obs_dim + kSacA, 2, hc, kSacA, 0, sh.critic))) return rc;          // fc1 -> fc2 -> fc_out
    sh.gld = sac_gld(c.hidden);
    return 0;
}

static size_t smem_target(const SacShape &s) { return (size_t)(s.actor.smem_total_floats + s.critic.smem_total_floats + s.critic.smem_w_floats + 3 * kTile * 32) * 4; }
static size_t smem_critic(const SacShape &s) { return (size_t)(s.critic.smem_total_floats + s.critic.smem_w_floats + 2 * kTile * s.gld + kTile * 32) * 4; }
static size_t smem_actor(const SacShape &s) { return (size_t)(s.actor.smem_total_floats + s.critic.smem_total_floats + s.critic.smem_w_floats + 2 * kTile * s.gld + 3 * kTile * 32) * 4; }
static size_t smem_act(const SacShape &s) { return (size_t)(s.actor.smem_total_floats + kTile * 32) * 4; }

// dynamic and static shared memory of one CTA of each kernel: target, critic, actor, act, and the weighted (prioritised-replay)
// critic, which adds its row weights, critic-1 outputs and loss sums to the critic's static shared memory
static int sac_smem_total(const SacShape &s, size_t out[5])
{
    const void *k[5] = { (const void *)sac_target_kernel<true>, (const void *)sac_critic_kernel<true, false>, (const void *)sac_actor_kernel<true>,
                         (const void *)sac_act_kernel<true>,      // the one-trainer instances declare the same static shared memory
                         (const void *)sac_critic_kernel<true, true> };
    const size_t dyn[5] = { smem_target(s), smem_critic(s), smem_actor(s), smem_act(s), smem_critic(s) };
    for (int i = 0; i < 5; ++i) {
        cudaFuncAttributes fa;
        UAVRL_CUDA(cudaFuncGetAttributes(&fa, k[i]));
        out[i] = dyn[i] + fa.sharedSizeBytes;
    }
    return 0;
}

// the kernels a learner of configuration c launches: their shared memory per block, *n of them (5 continuous, 4 discrete)
static int sac_smem_of(const uavrl_sac_config &c, const SacShape &s, size_t out[5], int *n)
{
    *n = c.discrete ? 4 : 5;
    return c.discrete ? sacd_smem_total(s, out) : sac_smem_total(s, out);
}

static int sac_pack(uavrl_sac *s, int role, cudaStream_t st)
{
    const NetDev &n = role == 0 ? s->sh.actor : s->sh.critic;
    pack_image_kernel<<<dim3((n.P + 255) / 256, s->G), 256, 0, st>>>(n.P, s->p[role], role == 0 ? s->map_a : s->map_c, s->img[role],
                                                                     n.smem_w_floats);
    UAVRL_LAUNCHED();
    return 0;
}

static void sac_fill_args(uavrl_sac *s, SacArgs &a, const BatchSrc &src, int B, int Bg, const float *eps, uint64_t ctr)
{
    memset(&a, 0, sizeof(a));
    a.actor = s->sh.actor; a.critic = s->sh.critic; a.src = src; a.B = B; a.Bg = Bg; a.n_tiles = (B + kTile - 1) / kTile; a.gld = s->sh.gld;
    a.img_actor = s->img[0]; a.img_c1 = s->img[1]; a.img_c2 = s->img[2]; a.img_t1 = s->img[3]; a.img_t2 = s->img[4];
    a.eps = eps; a.key = s->cfg.seed ^ kNoiseSalt; a.ctr = ctr; a.log_alpha = s->scal; a.td = s->td;
    a.part_a = s->part[0]; a.part_c1 = s->part[1]; a.part_c2 = s->part[2]; a.stat = s->stat;
    a.h = SacHyper{ s->cfg.actor_lr, s->cfg.critic_lr, s->cfg.alpha_lr, s->cfg.target_entropy, s->cfg.gamma, s->cfg.tau, s->cfg.action_bound };
}

static void adam_args(AdamArgs &a, const NetDev &n, int nparts, float lr, int64_t t)
{
    memset(&a, 0, sizeof(a));
    a.P = n.P; a.nparts = nparts; a.n_loss_parts = 0; a.apply = 1; a.world = 1; a.img_floats = n.smem_w_floats;
    adam_hyper(a, lr, t);
    a.inv_b = 1.f;
}

// the optimiser step of network r (0 actor, 1 and 2 the critics): no target network, no tensor-core images, no loss
static AdamPtrs sac_adam_ptrs(const uavrl_sac *s, int r)
{
    AdamPtrs q;
    memset(&q, 0, sizeof(q));
    q.partials = s->part[r]; q.loss_partials = s->lossbuf; q.grad = s->grad[r]; q.local = s->p[r]; q.m = s->m[r]; q.v = s->v[r];
    q.img_local = s->img[r]; q.img_map = r == 0 ? s->map_a : s->map_c;
    return q;
}

// gradient partial / stat slots per trainer for a per-trainer batch B: the tile kernels' grid.  They grow (never shrink) when a
// larger explicit batch arrives; TD targets likewise
static int sac_scratch(uavrl_sac *s, int B, int grid, cudaStream_t st)
{
    const size_t G = (size_t)s->G, Pa = (size_t)s->sh.actor.P, Pc = (size_t)s->sh.critic.P;
    if (int rc = grow(s->parts_mem, s->parts_cap, grid, st, true, buf(s->part[0], G * grid * Pa), buf(s->part[1], G * grid * Pc),
                      buf(s->part[2], G * grid * Pc), buf(s->stat, G * grid * 4)))
        return rc;
    return grow(s->td_mem, s->td_cap, B, st, true, buf(s->td, G * B * kSacA));
}

// the act kernel of every trainer on n rows (G equal blocks) with noise counter ctr, or the mean action
static int sac_act_launch(uavrl_sac *s, const float *obs, int n, const float *eps, uint64_t ctr, bool mean, float *actions,
                          cudaStream_t st)
{
    SacArgs a;
    BatchSrc none;
    memset(&none, 0, sizeof(none));
    const int ng = n / s->G;                                   // rows per trainer: block g belongs to trainer g
    sac_fill_args(s, a, none, ng, ng, eps, ctr);
    const int grid = a.n_tiles < s->max_ctas ? a.n_tiles : s->max_ctas;
    const size_t sm = smem_act(s->sh);
    if (mean && s->G > 1) sac_act_kernel<true, true><<<dim3(grid, s->G), kNetThreads, sm, st>>>(a, obs, ng, actions);
    else if (mean) sac_act_kernel<false, true><<<grid, kNetThreads, sm, st>>>(a, obs, ng, actions);
    else if (s->G > 1) sac_act_kernel<true><<<dim3(grid, s->G), kNetThreads, sm, st>>>(a, obs, ng, actions);
    else sac_act_kernel<false><<<grid, kNetThreads, sm, st>>>(a, obs, ng, actions);
    UAVRL_LAUNCHED();
    return 0;
}

int uavrl::launch_sac_act(uavrl_sac *s, const float *obs, int n, const float *eps, float *actions, cudaStream_t st)
{
    return sac_act_launch(s, obs, n, eps, 0x8000000000000000ull | s->calls++, false, actions, st);
}

int uavrl::launch_sac_act_eval(uavrl_sac *s, const float *obs, int n, bool mean, uint64_t ctr, float *actions, cudaStream_t st)
{
    return sac_act_launch(s, obs, n, nullptr, ctr, mean, actions, st);
}

// the discrete tile kernels' view of the learner: B rows per trainer, losses averaged over Bg rows
static void sacd_fill_args(uavrl_sac *s, SacdArgs &a, const BatchSrc &src, int B, int Bg)
{
    memset(&a, 0, sizeof(a));
    a.actor = s->sh.actor; a.critic = s->sh.critic; a.src = src; a.B = B; a.n_tiles = (B + kTile - 1) / kTile; a.gld = s->sh.gld;
    a.inv_b = 1.f / (float)Bg; a.gamma = s->cfg.gamma;
    a.img_actor = s->img[0]; a.img_c1 = s->img[1]; a.img_c2 = s->img[2]; a.img_t1 = s->img[3]; a.img_t2 = s->img[4];
    a.log_alpha = s->scal; a.td = s->td; a.part_a = s->part[0]; a.part_c1 = s->part[1]; a.part_c2 = s->part[2]; a.stat = s->stat;
    a.key = s->cfg.seed ^ kNoiseSalt; a.salt = kNoiseSalt;             // the continuous learner's noise stream convention
}

// the discrete act kernel of every trainer on n rows (G equal blocks) with draw counter ctr, or argmax p
static int sacd_act_launch(uavrl_sac *s, const float *obs, int n, const float *u, uint64_t ctr, bool mean, int32_t *actions, cudaStream_t st)
{
    BatchSrc none;
    memset(&none, 0, sizeof(none));
    const int ng = n / s->G;
    SacdArgs a;
    sacd_fill_args(s, a, none, ng, ng);
    a.ctr = ctr;
    return launch_sacd_act_kernel(a, obs, ng, u, mean, actions, a.n_tiles < s->max_ctas ? a.n_tiles : s->max_ctas, s->G, st);
}

int uavrl::launch_sacd_act(uavrl_sac *s, const float *obs, int n, const float *u, int32_t *actions, cudaStream_t st)
{
    return sacd_act_launch(s, obs, n, u, 0x8000000000000000ull | s->calls++, false, actions, st);
}

int uavrl::launch_sacd_act_eval(uavrl_sac *s, const float *obs, int n, bool mean, uint64_t ctr, int32_t *actions, cudaStream_t st)
{
    return sacd_act_launch(s, obs, n, nullptr, ctr, mean, actions, st);
}

static int sac_grid(const uavrl_sac *s, int B)
{
    const int n_tiles = (B + kTile - 1) / kTile;
    return n_tiles < s->max_ctas ? n_tiles : s->max_ctas;
}

// The update's first half on B rows per trainer (losses averaged over Bg rows): one Adam step counted, the TD targets, both
// critics' gradient partials and squared-error sums.  Prioritised replay (ReplayStore::per_samples): the batch is drawn from
// the trees first and src then reads through that sample, so the actor phase, given the same src, takes the same rows; the
// critic kernel weights its losses (any src with importance weights does) and its |errors| go back to the trees once it has run
static int sac_critic_phase(uavrl_sac *s, BatchSrc &src, int B, int Bg, const float *eps_next, cudaStream_t st)
{
    const int grid = sac_grid(s, B);
    int rc = sac_scratch(s, B, grid, st);
    if (rc) return rc;
    const bool per = s->replay.per_samples(src);
    if (per) {
        // the sample lives in the trees' scratch until the actor phase has read it
        if (s->dp_phase != 0) return fail(UAVRL_ERR_STATE, "a prioritised-replay update while a split update waits for its next phase");
        src = s->replay.per_source(s->cfg.seed, B, src, st, &rc);
        if (rc) return rc;
    }
    const dim3 tiles(grid, s->G);                        // y: trainer
    SacArgs a;
    s->adam_t += 1;
    sac_fill_args(s, a, src, B, Bg, eps_next, 2 * (uint64_t)s->epoch);
    if (s->G > 1) sac_target_kernel<true><<<tiles, kNetThreads, smem_target(s->sh), st>>>(a);
    else sac_target_kernel<false><<<grid, kNetThreads, smem_target(s->sh), st>>>(a);
    UAVRL_LAUNCHED();
    if (src.is_w) {
        if (s->G > 1) sac_critic_kernel<true, true><<<tiles, kNetThreads, smem_critic(s->sh), st>>>(a);
        else sac_critic_kernel<false, true><<<grid, kNetThreads, smem_critic(s->sh), st>>>(a);
    } else {
        if (s->G > 1) sac_critic_kernel<true, false><<<tiles, kNetThreads, smem_critic(s->sh), st>>>(a);
        else sac_critic_kernel<false, false><<<grid, kNetThreads, smem_critic(s->sh), st>>>(a);
    }
    UAVRL_LAUNCHED();
    return per ? s->replay.per_write_back(B, st) : 0;
}

// the second half, after the critics' step: the actor's gradient partials, loss and entropy sums on the same rows
static int sac_actor_phase(uavrl_sac *s, const BatchSrc &src, int B, int Bg, const float *eps_cur, cudaStream_t st)
{
    const int grid = sac_grid(s, B);
    SacArgs a;
    sac_fill_args(s, a, src, B, Bg, eps_cur, 2 * (uint64_t)s->epoch + 1);
    if (s->G > 1) sac_actor_kernel<true><<<dim3(grid, s->G), kNetThreads, smem_actor(s->sh), st>>>(a);
    else sac_actor_kernel<false><<<grid, kNetThreads, smem_actor(s->sh), st>>>(a);
    UAVRL_LAUNCHED();
    return 0;
}

// reduce_adam_kernel on network r (0 actor, 1 and 2 the critics): reduce the grid's partials and step (nparts > 0, apply),
// reduce only (apply false), or step on the gradient the caller all-reduced (nparts = 0)
static int sac_reduce_adam(uavrl_sac *s, int r, int nparts, bool apply, cudaStream_t st)
{
    AdamArgs aa;
    adam_args(aa, r == 0 ? s->sh.actor : s->sh.critic, nparts, r == 0 ? s->cfg.actor_lr : s->cfg.critic_lr, s->adam_t);
    aa.apply = apply ? 1 : 0;
    UAVRL_CUDA(launch_reduce_adam(s->G, st, false, aa, sac_adam_ptrs(s, r)));
    UAVRL_LAUNCHED();
    return 0;
}

// alpha step, soft target update and losses over Bg rows; exchanged: the stat sums are the exchange vectors' scalar words
static int sac_finish(uavrl_sac *s, int grid, int Bg, bool exchanged, float *losses_dev, cudaStream_t st)
{
    SacFinishArgs f;
    memset(&f, 0, sizeof(f));
    f.Pc = s->sh.critic.P; f.nparts = grid; f.img_floats = s->sh.critic.smem_w_floats;
    f.tau = s->cfg.tau; f.alpha_lr = s->cfg.alpha_lr; f.target_entropy = s->cfg.target_entropy;
    // continuous: every loss is a mean over B x action_dim; discrete: over the B rows (the entropy is one per row)
    f.inv_n = 1.f / ((float)Bg * (float)(s->cfg.discrete ? 1 : kSacA)); f.do_alpha = 1;
    AdamArgs aa;
    adam_hyper(aa, s->cfg.alpha_lr, s->adam_t);                    // the alpha step's bias corrections
    f.step_size_scale = aa.step_size; f.bc2_sqrt = aa.bc2_sqrt;
    const float *sums_c = exchanged ? s->xc + 2 * (size_t)s->sh.critic.P : nullptr, *sums_a = exchanged ? s->xa + s->sh.actor.P : nullptr;
    sac_finish_kernel<<<dim3((f.Pc + 255) / 256, s->G), 256, 0, st>>>(f, s->stat, sums_c, sums_a, s->scal, s->p[1], s->p[2], s->p[3], s->p[4],
                                                                     s->img[3], s->img[4], s->map_c, losses_dev ? losses_dev : s->out);
    UAVRL_LAUNCHED();
    return 0;
}

// The discrete update (SAC_Trainer.py:380-430): TD targets, both critics' gradients and Adam steps, then the actor on the
// updated critics and its Adam step, then the alpha step and the soft target update
static int sacd_update(uavrl_sac *s, const BatchSrc &src, int B, float *losses_dev, cudaStream_t st)
{
    const int grid = sac_grid(s, B);
    int rc = sac_scratch(s, B, grid, st);
    if (rc) return rc;
    s->adam_t += 1;
    SacdArgs a;
    sacd_fill_args(s, a, src, B, B);
    if ((rc = launch_sacd_phase(kSacdTarget, a, grid, s->G, st)) || (rc = launch_sacd_phase(kSacdCritic, a, grid, s->G, st)) ||
        (rc = sac_reduce_adam(s, 1, grid, true, st)) || (rc = sac_reduce_adam(s, 2, grid, true, st)) ||
        (rc = launch_sacd_phase(kSacdActor, a, grid, s->G, st)) || (rc = sac_reduce_adam(s, 0, grid, true, st)))
        return rc;
    return sac_finish(s, grid, B, false, losses_dev, st);
}

int uavrl::launch_sac_update(uavrl_sac *s, const BatchSrc &src_in, int B, const float *eps_next, const float *eps_cur, float *losses_dev,
                             cudaStream_t st)
{
    if (s->cfg.discrete) return sacd_update(s, src_in, B, losses_dev, st);
    const int grid = sac_grid(s, B);
    BatchSrc src = src_in;
    int rc;
    if ((rc = sac_critic_phase(s, src, B, B, eps_next, st)) || (rc = sac_reduce_adam(s, 1, grid, true, st)) ||
        (rc = sac_reduce_adam(s, 2, grid, true, st)) || (rc = sac_actor_phase(s, src, B, B, eps_cur, st)) ||
        (rc = sac_reduce_adam(s, 0, grid, true, st)))
        return rc;
    return sac_finish(s, grid, B, false, losses_dev, st);
}

// One fused exchange (dp_allreduce_adam_kernel) of this rank's gradients and stat sums: critics = both critics' gradients and
// squared-error sums into xc, else the actor's gradient and its loss / entropy sums into xa; then Adam on those networks
static int sac_exchange(uavrl_sac *s, bool critics, int grid, cudaStream_t st)
{
    const NetDev &n = critics ? s->sh.critic : s->sh.actor;
    AdamArgs aa;
    adam_args(aa, n, grid, critics ? s->cfg.critic_lr : s->cfg.actor_lr, s->adam_t);
    aa.world = s->comm.world;
    DpExchange x;
    memset(&x, 0, sizeof(x));
    x.n_seg = critics ? 2 : 1;
    for (int k = 0; k < x.n_seg; ++k) {
        const int r = critics ? 1 + k : 0;
        x.seg[k].partials = s->part[r]; x.seg[k].nparts = grid; x.seg[k].P = n.P;
        x.seg[k].q = sac_adam_ptrs(s, r);
    }
    x.extra_parts = s->stat + (critics ? 0 : 2); x.n_extra_parts = grid; x.extra_stride = 4; x.n_extra = 2; x.extra_scale = 1.f;
    x.extra_out = critics ? s->xc + 2 * (size_t)n.P : s->xa + n.P;
    UAVRL_CUDA(launch_dp_exchange(s->comm, aa, x, st, false));
    UAVRL_LAUNCHED();
    return 0;
}

int uavrl::launch_sac_update_dp(uavrl_sac *s, const BatchSrc &src_in, int B, int global_batch, const float *eps_next, const float *eps_cur,
                                float *losses_dev, cudaStream_t st)
{
    const int grid = sac_grid(s, B);
    BatchSrc src = src_in;
    int rc;
    if ((rc = sac_critic_phase(s, src, B, global_batch, eps_next, st)) || (rc = sac_exchange(s, true, grid, st)) ||
        (rc = sac_actor_phase(s, src, B, global_batch, eps_cur, st)) || (rc = sac_exchange(s, false, grid, st)))
        return rc;
    return sac_finish(s, grid, global_batch, true, losses_dev, st);
}

// everything a learner allocates; on failure the caller destroys the half-built handle
static int sac_alloc(uavrl_sac *s)
{
    const uavrl_sac_config *cfg = &s->cfg;
    const size_t G = (size_t)s->G;
    DevMem &mem = s->mem;
    int rc;
    for (int r = 0; r < 5; ++r) {
        const NetDev &n = r == 0 ? s->sh.actor : s->sh.critic;
        if ((rc = mem.alloc(s->p[r], G * n.P)) || (rc = mem.alloc(s->img[r], G * n.smem_w_floats))) return rc;
    }
    for (int r = 0; r < 3; ++r) {
        const NetDev &n = r == 0 ? s->sh.actor : s->sh.critic;
        if ((rc = mem.alloc(s->m[r], G * n.P)) || (rc = mem.alloc(s->v[r], G * n.P))) return rc;
    }
    const size_t Pa = (size_t)s->sh.actor.P, Pc = (size_t)s->sh.critic.P;
    if ((rc = mem.alloc(s->xa, G * Pa + 2)) || (rc = mem.alloc(s->xc, 2 * G * Pc + 2))) return rc;
    s->grad[0] = s->xa; s->grad[1] = s->xc; s->grad[2] = s->xc + G * Pc;
    std::vector<int32_t> ma, mc;
    build_image_map(s->sh.actor, ma); build_image_map(s->sh.critic, mc);
    if ((rc = mem.alloc(s->map_a, ma.size())) || (rc = mem.alloc(s->map_c, mc.size()))) return rc;
    UAVRL_CUDA(cudaMemcpy(s->map_a, ma.data(), ma.size() * 4, cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(s->map_c, mc.data(), mc.size() * 4, cudaMemcpyHostToDevice));
    if ((rc = sac_scratch(s, cfg->batch_size, trainer_parts_cap(s->G, cfg->batch_size, s->max_ctas), 0))) return rc;
    if ((rc = mem.alloc(s->scal, 3 * G)) || (rc = mem.alloc(s->out, 4 * G)) || (rc = mem.alloc(s->lossbuf, 1))) return rc;
    std::vector<float> init(3 * G, 0.f);
    for (size_t g = 0; g < G; ++g) init[3 * g] = logf(0.01f);          // SAC_Trainer.py:53
    UAVRL_CUDA(cudaMemcpy(s->scal, init.data(), init.size() * 4, cudaMemcpyHostToDevice));
    // the ring holds float[2] actions (continuous) or int32 action indices (discrete)
    if (cfg->lockstep_envs > 0 && (rc = s->replay.alloc(cfg->replay_capacity, cfg->lockstep_envs, s->G, cfg->obs_dim, !cfg->discrete))) return rc;
    if (cfg->discrete) return sacd_raise_smem(s->sh);
    if ((rc = raise_dyn_smem(sac_target_kernel<false>, smem_target(s->sh))) || (rc = raise_dyn_smem(sac_critic_kernel<false, false>, smem_critic(s->sh))) ||
        (rc = raise_dyn_smem(sac_actor_kernel<false>, smem_actor(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<false>, smem_act(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<false, true>, smem_act(s->sh))) ||
        (rc = raise_dyn_smem(sac_target_kernel<true>, smem_target(s->sh))) || (rc = raise_dyn_smem(sac_critic_kernel<true, false>, smem_critic(s->sh))) ||
        (rc = raise_dyn_smem(sac_actor_kernel<true>, smem_actor(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<true>, smem_act(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<true, true>, smem_act(s->sh))) ||
        (rc = raise_dyn_smem(sac_critic_kernel<false, true>, smem_critic(s->sh))) || (rc = raise_dyn_smem(sac_critic_kernel<true, true>, smem_critic(s->sh))))
        return rc;
    return 0;
}

// entry points of one action kind only (`what` names the call): refused before anything is enqueued or allocated
static int refuse_discrete(const uavrl_sac *s, const std::string &what)
{
    if (s->cfg.discrete) return fail(UAVRL_ERR_INVALID, what + " is not available on a discrete SAC learner");
    return 0;
}
static int refuse_continuous(const uavrl_sac *s, const std::string &what)
{
    if (!s->cfg.discrete) return fail(UAVRL_ERR_INVALID, what + " needs a discrete SAC learner (discrete = 1)");
    return 0;
}

extern "C" {

int uavrl_sac_smem_bytes(const uavrl_sac_config *cfg, int64_t *bytes_out)
{
    if (!cfg || !bytes_out) return fail(UAVRL_ERR_INVALID, "uavrl_sac_smem_bytes: null argument");
    SacShape sh;
    int rc = sac_shape(*cfg, sh);
    if (rc) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(UAVRL_ERR_CUDA, "no CUDA device: the SAC learner has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg->device));
    size_t b[5];
    int nk;
    if ((rc = sac_smem_of(*cfg, sh, b, &nk))) return rc;
    for (int i = 0; i < 4; ++i) bytes_out[i] = (int64_t)b[i];
    return 0;
}

int uavrl_sac_create(const uavrl_sac_config *cfg, uavrl_sac **out)
{
    return uavrl_sac_create_trainers(cfg, 1, out);
}

int uavrl_sac_create_trainers(const uavrl_sac_config *cfg, int32_t n_trainers, uavrl_sac **out)
{
    if (!cfg || !out) return fail(UAVRL_ERR_INVALID, "uavrl_sac_create: null argument");
    SacShape sh;
    int rc = sac_shape(*cfg, sh);
    if (rc || (rc = check_trainer_group(*cfg, n_trainers, "SAC learner"))) return rc;
    size_t smem[5];
    int nk;
    if ((rc = sac_smem_of(*cfg, sh, smem, &nk))) return rc;
    for (int i = 0; i < nk; ++i)
        if (smem[i] > kMaxBlockSmem)
            return fail(UAVRL_ERR_INVALID, "networks too large for the SMEM-resident SAC kernels: " + std::to_string(smem[i]) +
                                               " B of shared memory per block, at most " + std::to_string(kMaxBlockSmem));
    uavrl_sac *s = new uavrl_sac();
    s->cfg = *cfg;
    s->sh = sh;
    s->G = n_trainers;
    {   // grid cap of the tile kernels: 4 CTAs per SM's worth of tiles, i.e. one tile per CTA up to batch 4 x SMs x 32.  (One CTA
        // per SM looping over its tiles would accumulate ONE partial, at the price of a read-modify-write of the global partial
        // per tile.)
        const char *ov = getenv("UAVRL_SAC_MAX_CTAS");            // tests: force the multi-tile (accumulating) path on a small batch
        if (ov && atoi(ov) > 0) s->max_ctas = atoi(ov);
    }
    if ((rc = sac_alloc(s))) {
        uavrl_sac_destroy(s);
        return rc;
    }
    *out = s;
    return 0;
}

int uavrl_sac_destroy(uavrl_sac *s)
{
    if (!s) return 0;
    cudaSetDevice(s->cfg.device);
    cudaDeviceSynchronize();
    delete s;
    return 0;
}

int64_t uavrl_sac_param_count(const uavrl_sac *s, int32_t role) { return !s ? 0 : (role == 0 ? s->sh.actor.P : s->sh.critic.P); }
int32_t uavrl_sac_trainer_count(const uavrl_sac *s) { return s ? s->G : 0; }

static float *sac_buf(uavrl_sac *s, int role)
{
    if (role >= 0 && role < 5) return s->p[role];
    if (role >= 5 && role < 8) return s->m[role - 5];
    if (role >= 8 && role < 11) return s->v[role - 8];
    if (role >= 11 && role < 14) return s->grad[role - 11];        // last reduced gradients: read-only
    return nullptr;
}

int uavrl_sac_set_params(uavrl_sac *s, int32_t role, const float *h)
{
    if (!s || !h || !sac_buf(s, role)) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (role >= 11) return fail(UAVRL_ERR_INVALID, "roles 11-13 (the last reduced gradients) are read-only");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const int rr = role < 5 ? role : (role - 5) % 3;
    const int P = rr == 0 ? s->sh.actor.P : s->sh.critic.P;
    UAVRL_CUDA(cudaMemcpy(sac_buf(s, role), h, (size_t)s->G * P * 4, cudaMemcpyHostToDevice));
    if (role < 5) { int rc = sac_pack(s, role, 0); if (rc) return rc; UAVRL_CUDA(cudaDeviceSynchronize()); }
    return 0;
}

int uavrl_sac_get_params(uavrl_sac *s, int32_t role, float *h)
{
    if (!s || !h || !sac_buf(s, role)) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const int rr = role < 5 ? role : (role - 5) % 3;
    const int P = rr == 0 ? s->sh.actor.P : s->sh.critic.P;
    UAVRL_CUDA(cudaMemcpy(h, sac_buf(s, role), (size_t)s->G * P * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_sac_set_alpha(uavrl_sac *s, const float *h)
{
    if (!s || !h) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(s->scal, h, (size_t)s->G * 3 * 4, cudaMemcpyHostToDevice));
    return 0;
}

int uavrl_sac_get_alpha(uavrl_sac *s, float *h)
{
    if (!s || !h) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    UAVRL_CUDA(cudaMemcpy(h, s->scal, (size_t)s->G * 3 * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_sac_set_scalars(uavrl_sac *s, float log_alpha, float la_m, float la_v, int64_t epoch, int64_t adam_step)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    std::vector<float> v((size_t)s->G * 3);                    // the same triple for every trainer
    for (size_t g = 0; g < (size_t)s->G; ++g) { v[3 * g] = log_alpha; v[3 * g + 1] = la_m; v[3 * g + 2] = la_v; }
    UAVRL_CUDA(cudaMemcpy(s->scal, v.data(), v.size() * 4, cudaMemcpyHostToDevice));
    s->epoch = epoch; s->adam_t = adam_step;
    return 0;
}

int uavrl_sac_get_scalars(uavrl_sac *s, float *log_alpha, float *la_m, float *la_v, int64_t *epoch, int64_t *adam_step)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    float v[3];
    UAVRL_CUDA(cudaMemcpy(v, s->scal, sizeof(v), cudaMemcpyDeviceToHost));
    if (log_alpha) *log_alpha = v[0];
    if (la_m) *la_m = v[1];
    if (la_v) *la_v = v[2];
    if (epoch) *epoch = s->epoch;
    if (adam_step) *adam_step = s->adam_t;
    return 0;
}

int uavrl_sac_act(uavrl_sac *s, const float *obs_dev, int32_t n, const float *eps_dev, float *actions_dev, void *stream)
{
    if (!s || !obs_dev || !actions_dev || n <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_discrete(s, "uavrl_sac_act (use uavrl_sac_act_discrete)")) return rc;
    if (n % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_act: n must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    return launch_sac_act(s, obs_dev, n, eps_dev, actions_dev, (cudaStream_t)stream);
}

int uavrl_sac_act_discrete(uavrl_sac *s, const float *obs_dev, int32_t n, const float *u_dev, int32_t mean_action, int32_t *actions_dev,
                           void *stream)
{
    if (!s || !obs_dev || !actions_dev || n <= 0 || (mean_action != 0 && mean_action != 1)) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_continuous(s, "uavrl_sac_act_discrete")) return rc;
    if (n % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_act_discrete: n must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    if (mean_action) return launch_sacd_act_eval(s, obs_dev, n, true, 0, actions_dev, (cudaStream_t)stream);
    return launch_sacd_act(s, obs_dev, n, u_dev, actions_dev, (cudaStream_t)stream);
}

int uavrl_sac_act_mean(uavrl_sac *s, const float *obs_dev, int32_t n, float *actions_dev, void *stream)
{
    if (!s || !obs_dev || !actions_dev || n <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_discrete(s, "uavrl_sac_act_mean (use uavrl_sac_act_discrete with mean_action = 1)")) return rc;
    if (n % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_act_mean: n must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    return launch_sac_act_eval(s, obs_dev, n, true, 0, actions_dev, (cudaStream_t)stream);
}

// a_dev: float [B][2] (continuous) or int32 [B] (discrete)
static BatchSrc sac_explicit_src(const uavrl_sac *s, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                                 const float *d_dev)
{
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kBatchExplicit; src.frames = s_dev; src.s2_rows = s2_dev; src.rew = r_dev; src.done_f32 = d_dev;
    if (s->cfg.discrete) src.act = reinterpret_cast<const int32_t *>(a_dev);
    else src.act2 = a_dev;
    return src;
}

int uavrl_sac_update_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                           const float *d_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev, void *stream)
{
    if (!s || B <= 0 || !s_dev || !a_dev || !r_dev || !s2_dev || !d_dev) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (B % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_update_batch: B must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    return launch_sac_update(s, sac_explicit_src(s, s_dev, a_dev, r_dev, s2_dev, d_dev), B / s->G, eps_next_dev, eps_cur_dev, losses_dev,
                             (cudaStream_t)stream);
}

int uavrl_sac_update_batch_per(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                               const float *d_dev, const float *is_weights_dev, float *abs_err_out_dev, const float *eps_next_dev,
                               const float *eps_cur_dev, float *losses_dev, void *stream)
{
    if (!s || B <= 0 || !s_dev || !a_dev || !r_dev || !s2_dev || !d_dev || !is_weights_dev) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_discrete(s, "uavrl_sac_update_batch_per (prioritised replay)")) return rc;
    if (B % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_update_batch_per: B must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    BatchSrc src = sac_explicit_src(s, s_dev, a_dev, r_dev, s2_dev, d_dev);
    src.is_w = is_weights_dev; src.abs_err = abs_err_out_dev;
    return launch_sac_update(s, src, B / s->G, eps_next_dev, eps_cur_dev, losses_dev, (cudaStream_t)stream);
}

int64_t uavrl_sac_replay_size(const uavrl_sac *s) { return s ? s->replay.count : 0; }

int uavrl_sac_replay_gather(uavrl_sac *s, int32_t n, const int64_t *idx, float *s_host, float *a_host, float *r_host, float *s2_host,
                            uint8_t *d_host)
{
    if (!s || n <= 0 || !idx) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (!s->replay.frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    if (s->cfg.discrete) return s->replay.gather(n, idx, s_host, reinterpret_cast<int32_t *>(a_host), nullptr, r_host, s2_host, d_host);
    return s->replay.gather(n, idx, s_host, nullptr, a_host, r_host, s2_host, d_host);
}

int uavrl_sac_update_replay(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev,
                            void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (!s->replay.frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    if (!s->replay.ready(s->cfg.batch_size)) return 0;         // nothing sampled yet
    return launch_sac_update(s, s->replay.source(s->cfg.seed, s->epoch, idx_tape_dev), s->cfg.batch_size, eps_next_dev, eps_cur_dev,
                             losses_dev, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ prioritised replay: one SumTree per trainer over its slots
// of the lockstep ring (ReplayStore::per, per.cu); the updates that sample the ring use them once enabled
int uavrl_sac_per_enable(uavrl_sac *s, double alpha, double beta0, double beta_inc, double eps, double err_upper)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = refuse_discrete(s, "uavrl_sac_per_enable (prioritised replay)")) return rc;
    if (!s->replay.frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    return s->replay.per_enable(alpha, beta0, beta_inc, eps, err_upper);
}

int uavrl_sac_per_set_priorities(uavrl_sac *s, int32_t n, const int32_t *slots_dev, const double *prio_dev, void *stream)
{
    return per_entry_set(s ? &s->replay : nullptr, s ? s->cfg.device : 0, n, slots_dev, prio_dev, nullptr, 0, (cudaStream_t)stream);
}

int uavrl_sac_per_set_errors(uavrl_sac *s, int32_t n, const int32_t *slots_dev, const float *abs_err_dev, int32_t clip, void *stream)
{
    return per_entry_set(s ? &s->replay : nullptr, s ? s->cfg.device : 0, n, slots_dev, nullptr, abs_err_dev, clip, (cudaStream_t)stream);
}

int uavrl_sac_per_sample(uavrl_sac *s, int32_t B, const double *u_tape_dev, int32_t *slots_out_dev, float *weights_out_dev, void *stream)
{
    // a larger B regrows the trees' scratch, which a waiting split update still reads its rows through
    if (s && s->dp_phase != 0) return fail(UAVRL_ERR_STATE, "uavrl_sac_per_sample while a split update waits for its next phase");
    return per_entry_sample(s ? &s->replay : nullptr, s ? s->cfg.device : 0, s ? s->cfg.seed : 0, B, u_tape_dev, slots_out_dev,
                            weights_out_dev, (cudaStream_t)stream);
}

int uavrl_sac_per_get(uavrl_sac *s, double *leaves_host, double *total_out, double *beta_out)
{
    return per_entry_get(s ? &s->replay : nullptr, s ? s->cfg.device : 0, leaves_host, total_out, beta_out);
}

int uavrl_sac_federate_actors(uavrl_sac *s, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int P = s->sh.actor.P;
    sac_federate_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, s->G, s->p[0], s->G, s->p[0]);
    UAVRL_LAUNCHED();
    return sac_pack(s, 0, st);                                 // the G actor images
}

int uavrl_sac_fed_shard(uavrl_sac *s, int32_t rank, int32_t world)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (world < 1 || rank < 0 || rank >= world) return fail(UAVRL_ERR_INVALID, "uavrl_sac_fed_shard: needs world >= 1 and rank in [0, world)");
    const int64_t G = (int64_t)s->G * world;
    if (G > 65535) return fail(UAVRL_ERR_INVALID, "uavrl_sac_fed_shard: the global trainer count (trainers x world) must be at most 65535");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    DevMem mem;
    float *x = nullptr;
    if (int rc = mem.alloc(x, (size_t)G * s->sh.actor.P, false)) return rc;
    s->fed_mem = std::move(mem);
    s->fed_x = x; s->fed_rank = rank; s->fed_world = world; s->fed_phase = 0;
    return 0;
}

float *uavrl_sac_fed_exchange_ptr(uavrl_sac *s, int64_t *len_out)
{
    if (!s || !s->fed_world) return nullptr;
    if (len_out) *len_out = (int64_t)s->G * s->fed_world * s->sh.actor.P;
    return s->fed_x;
}

int uavrl_sac_fed_local(uavrl_sac *s, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (!s->fed_world) return fail(UAVRL_ERR_STATE, "uavrl_sac_fed_local before uavrl_sac_fed_shard");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const size_t P = s->sh.actor.P, GL = s->G;
    UAVRL_CUDA(cudaMemcpyAsync(s->fed_x + (size_t)s->fed_rank * GL * P, s->p[0], GL * P * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    s->fed_phase = 1;
    return 0;
}

int uavrl_sac_federate_actors_sharded(uavrl_sac *s, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (!s->fed_world) return fail(UAVRL_ERR_STATE, "uavrl_sac_federate_actors_sharded before uavrl_sac_fed_shard");
    if (s->fed_phase != 1)
        return fail(UAVRL_ERR_STATE, "uavrl_sac_federate_actors_sharded called out of order: it runs after uavrl_sac_fed_local and the gather");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int P = s->sh.actor.P;
    sac_federate_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, s->G * s->fed_world, s->fed_x, s->G, s->p[0]);
    UAVRL_LAUNCHED();
    s->fed_phase = 0;
    return sac_pack(s, 0, st);
}


// ------------------------------------------------------------------ data-parallel training
// the refusals every data-parallel update makes before its epoch counts
static int sac_dp_checks(const uavrl_sac *s, int32_t global_batch, bool ring, const char *fn)
{
    if (int rc = refuse_discrete(s, fn)) return rc;
    if (int rc = refuse_grouped(s->G, fn)) return rc;
    if (global_batch <= 0) return fail(UAVRL_ERR_INVALID, std::string(fn) + ": global_batch must be > 0");
    if (s->dp_phase != 0) return fail(UAVRL_ERR_STATE, std::string(fn) + " while a split update waits for its next phase");
    if (ring && !s->replay.frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    // every rank must take part in every exchange, and a rank that retries stays on the other ranks' sample keys
    if (ring && !s->replay.ready(s->cfg.batch_size)) return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions");
    return 0;
}

int uavrl_sac_comm_init(uavrl_sac *s, int32_t rank, int32_t world, void *handle_out)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "bad rank/world/handle pointer");
    if (int rc = refuse_discrete(s, "uavrl_sac_comm_init")) return rc;
    if (int rc = refuse_grouped(s->G, "uavrl_sac_comm_init")) return rc;
    const size_t Pa = (size_t)s->sh.actor.P, Pc = (size_t)s->sh.critic.P;
    return comm_init(s->comm, s->cfg.device, rank, world, 2 * Pc + 2 > Pa + 2 ? 2 * Pc + 2 : Pa + 2, handle_out, true);
}

int uavrl_sac_comm_connect(uavrl_sac *s, const void *handles)
{
    if (!s || !handles) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = refuse_discrete(s, "uavrl_sac_comm_connect")) return rc;
    if (int rc = refuse_grouped(s->G, "uavrl_sac_comm_connect")) return rc;
    if (!s->comm.recv) return fail(UAVRL_ERR_STATE, "uavrl_sac_comm_connect before uavrl_sac_comm_init");
    return comm_connect(s->comm, s->cfg.device, handles, true);
}

int uavrl_sac_update_replay_dp(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, const float *eps_cur_dev,
                               int32_t global_batch, float *losses_dev, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = sac_dp_checks(s, global_batch, true, "uavrl_sac_update_replay_dp")) return rc;
    if (!s->comm.ready) return fail(UAVRL_ERR_STATE, "uavrl_sac_update_replay_dp before uavrl_sac_comm_connect");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    return launch_sac_update_dp(s, s->replay.source(s->cfg.seed, s->epoch, idx_tape_dev), s->cfg.batch_size, global_batch, eps_next_dev,
                                eps_cur_dev, losses_dev, (cudaStream_t)stream);
}

// the split form's critic phase on src: the critics' gradients and squared-error sums into the critic exchange vector
static int sac_split_critic(uavrl_sac *s, const BatchSrc &src, int B, int global_batch, const float *eps_next, cudaStream_t st)
{
    s->dp_src = src; s->dp_B = B; s->dp_global = global_batch;           // the critic phase points dp_src at a prioritised sample
    const int grid = sac_grid(s, B);
    int rc;
    if ((rc = sac_critic_phase(s, s->dp_src, B, global_batch, eps_next, st)) || (rc = sac_reduce_adam(s, 1, grid, false, st)) ||
        (rc = sac_reduce_adam(s, 2, grid, false, st)))
        return rc;
    sac_stat_sums_kernel<<<1, 32, 0, st>>>(s->stat, grid, 0, s->xc + 2 * (size_t)s->sh.critic.P);
    UAVRL_LAUNCHED();
    s->dp_phase = 1;
    return 0;
}

int uavrl_sac_critic_grads_replay(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, int32_t global_batch, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = sac_dp_checks(s, global_batch, true, "uavrl_sac_critic_grads_replay")) return rc;
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;
    return sac_split_critic(s, s->replay.source(s->cfg.seed, s->epoch, idx_tape_dev), s->cfg.batch_size, global_batch, eps_next_dev,
                            (cudaStream_t)stream);
}

int uavrl_sac_critic_grads_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                                 const float *d_dev, const float *eps_next_dev, int32_t global_batch, void *stream)
{
    if (!s || B <= 0 || !s_dev || !a_dev || !r_dev || !s2_dev || !d_dev) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (int rc = sac_dp_checks(s, global_batch, false, "uavrl_sac_critic_grads_batch")) return rc;
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;
    return sac_split_critic(s, sac_explicit_src(s, s_dev, a_dev, r_dev, s2_dev, d_dev), B, global_batch, eps_next_dev, (cudaStream_t)stream);
}

static int sac_phase_is(const uavrl_sac *s, int phase, const char *fn)
{
    if (int rc = refuse_discrete(s, fn)) return rc;
    if (int rc = refuse_grouped(s->G, fn)) return rc;
    static const char *want[4] = { "", "after uavrl_sac_critic_grads_*", "after uavrl_sac_apply_critic_grads", "after uavrl_sac_actor_grads" };
    if (s->dp_phase != phase) return fail(UAVRL_ERR_STATE, std::string(fn) + " called out of order: it runs " + want[phase]);
    return 0;
}

int uavrl_sac_apply_critic_grads(uavrl_sac *s, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = sac_phase_is(s, 1, "uavrl_sac_apply_critic_grads")) return rc;
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if ((rc = sac_reduce_adam(s, 1, 0, true, st)) || (rc = sac_reduce_adam(s, 2, 0, true, st))) return rc;
    s->dp_phase = 2;
    return 0;
}

int uavrl_sac_actor_grads(uavrl_sac *s, const float *eps_cur_dev, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = sac_phase_is(s, 2, "uavrl_sac_actor_grads")) return rc;
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int grid = sac_grid(s, s->dp_B);
    int rc;
    if ((rc = sac_actor_phase(s, s->dp_src, s->dp_B, s->dp_global, eps_cur_dev, st)) || (rc = sac_reduce_adam(s, 0, grid, false, st)))
        return rc;
    sac_stat_sums_kernel<<<1, 32, 0, st>>>(s->stat, grid, 2, s->xa + s->sh.actor.P);
    UAVRL_LAUNCHED();
    s->dp_phase = 3;
    return 0;
}

int uavrl_sac_apply_actor_grads(uavrl_sac *s, float *losses_dev, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (int rc = sac_phase_is(s, 3, "uavrl_sac_apply_actor_grads")) return rc;
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if ((rc = sac_reduce_adam(s, 0, 0, true, st)) || (rc = sac_finish(s, sac_grid(s, s->dp_B), s->dp_global, true, losses_dev, st))) return rc;
    s->dp_phase = 0;
    return 0;
}

float *uavrl_sac_exchange_ptr(uavrl_sac *s, int32_t phase, int64_t *len_out)
{
    if (!s || (phase != 0 && phase != 1)) return nullptr;
    if (len_out) *len_out = phase == 0 ? 2 * (int64_t)s->sh.critic.P + 2 : (int64_t)s->sh.actor.P + 2;
    return phase == 0 ? s->xc : s->xa;
}

}  // extern "C"
