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
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "env.cuh"
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
template <bool GR>
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
    if (threadIdx.x == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) { stage_weights(cn, sac_img<GR>(a.img_c1, cn), RC, &bar[0]); stage_weights(cn, sac_img<GR>(a.img_c2, cn), WC2, &bar[1]); }
    uint32_t pkey[4];
    Philox::gen(sac_sample_key<GR>(a), a.src.epoch, 0x5A17ull, pkey);
    const float inv = 1.f / ((float)a.B * (float)kSacA);
    float sq[2] = { 0.f, 0.f };
    bool ready = false;
    int iter = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr; tr.ax = tr.ay = 0.f;
            if (gb < a.B) tr = resolve_transition(sac_src<GR>(a), gb, cn.in_dim - kSacA, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr; s_act[threadIdx.x][0] = tr.ax; s_act[threadIdx.x][1] = tr.ay;
        }
        __syncthreads();
        load_rows(rows, dYa, gld * 2, cn.in_dim - kSacA);                   // stage s in the (still unused) gradient planes: 32 x 2 gld
        __syncthreads();
        build_critic_input(dYa, gld * 2, cn.in_dim - kSacA, RC + cn.act_off[0], cn.act_ld[0], s_act);
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
                if (gb < a.B)
                    for (int j = 0; j < kSacA; ++j) {
                        const float diff = Q[b * 32 + j] - sac_td<GR>(a)[(size_t)gb * kSacA + j];
                        e2 += diff * diff;
                        g[j] = 2.f * diff * inv;
                    }
                s_sq[b] = e2;
            }
            __syncthreads();
            if (threadIdx.x == 0) { float s = 0.f; for (int b = 0; b < kTile; ++b) s += s_sq[b]; sq[which] += s; }
            critic_backward_tile(cn, sw, RC, dYa, dYb, gld, (which ? a.part_c2 : a.part_c1) + sac_part<GR>() * cn.P, iter > 0, nullptr, 0);
        }
    }
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
    const float inv = 1.f / ((float)a.B * (float)kSacA);
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

// blockIdx.y = trainer g: its stat [nparts][4], scal [3], critics and targets [Pc], target images and out [4]
__global__ void sac_finish_kernel(SacFinishArgs f, const float *__restrict__ stat, float *__restrict__ scal, const float *__restrict__ c1,
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
        // chain of dependent global loads)
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (int c = threadIdx.x; c < f.nparts; c += 32) {
            const float4 t = *reinterpret_cast<const float4 *>(stat + 4 * c);
            s0 += t.x; s1 += t.y; s2 += t.z; s3 += t.w;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, off); s1 += __shfl_xor_sync(0xffffffffu, s1, off);
            s2 += __shfl_xor_sync(0xffffffffu, s2, off); s3 += __shfl_xor_sync(0xffffffffu, s3, off);
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

// get_action (:444-448): action = actor(state)[0] with fresh noise.  Trainer blockIdx.y acts for rows [g n, (g + 1) n).
template <bool GR>
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
            if (gb < n) {
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
// float32 sum theta_0 + theta_1 + ... + theta_{G-1}, added left to right in trainer order.  One thread per actor parameter.
__global__ void sac_federate_kernel(int P, int G, float *__restrict__ actor)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float s = actor[i];
    for (int g = 1; g < G; ++g) s = __fadd_rn(s, actor[(size_t)g * P + i]);
    for (int g = 0; g < G; ++g) actor[(size_t)g * P + i] = s;
}

// uavrl_sac_replay_gather: logical indices of the lockstep ring -> packed rows (one warp per transition)
__global__ void sac_gather_kernel(int n, int in, BatchSrc src, const int64_t *__restrict__ idx, float *__restrict__ s, float *__restrict__ s2,
                                  float *__restrict__ a, float *__restrict__ r, uint8_t *__restrict__ d)
{
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n) return;
    const int64_t j = idx[i];
    const int64_t f = (src.oldest + j / src.n_envs) % src.cap, e = j % src.n_envs;
    const int64_t slot = f * src.n_envs + e, slot2 = ((f + 1) % src.cap) * src.n_envs + e;
    for (int k = lane; k < in; k += 32) {
        if (s) s[(size_t)i * in + k] = src.frames[(size_t)slot * in + k];
        if (s2) s2[(size_t)i * in + k] = src.frames[(size_t)slot2 * in + k];
    }
    if (lane == 0) {
        if (a) { a[2 * i] = src.act2[2 * slot]; a[2 * i + 1] = src.act2[2 * slot + 1]; }
        if (r) r[i] = src.rew[slot];
        if (d) d[i] = src.done_u8[slot];
    }
}

}  // namespace uavrl

using namespace uavrl;

// ------------------------------------------------------------------ host handle
// the two networks of a SAC learner and the stride of its gradient planes: everything the kernels' shared memory follows from
struct SacShape { NetDev actor, critic; int32_t gld; };

constexpr size_t kSacMaxSmem = 227 * 1024;     // shared memory one block may use on sm_90

// refuses a configuration before anything is allocated
static int sac_shape(const uavrl_sac_config &c, SacShape &sh)
{
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

// dynamic and static shared memory of one CTA of each kernel: target, critic, actor, act
static int sac_smem_total(const SacShape &s, size_t out[4])
{
    const void *k[4] = { (const void *)sac_target_kernel<true>, (const void *)sac_critic_kernel<true>, (const void *)sac_actor_kernel<true>,
                         (const void *)sac_act_kernel<true> };     // the one-trainer instances declare the same static shared memory
    const size_t dyn[4] = { smem_target(s), smem_critic(s), smem_actor(s), smem_act(s) };
    for (int i = 0; i < 4; ++i) {
        cudaFuncAttributes fa;
        UAVRL_CUDA(cudaFuncGetAttributes(&fa, k[i]));
        out[i] = dyn[i] + fa.sharedSizeBytes;
    }
    return 0;
}

// A grouped learner (uavrl_sac_create_trainers) holds G trainers: every per-network vector, weight image and scratch array
// below is [G][...]; trainer g acts for envs [g Ng, (g + 1) Ng) of the shared ring frames and samples only their transitions.
struct uavrl_sac {
    uavrl_sac_config cfg;
    SacShape sh;
    int32_t G = 1;
    float *p[5] = { nullptr }, *img[5] = { nullptr };      // actor, c1, c2, t1, t2
    float *m[3] = { nullptr }, *v[3] = { nullptr }, *grad[3] = { nullptr };
    int32_t *map_a = nullptr, *map_c = nullptr;
    float *part[3] = { nullptr };                          // gradient partials [G][parts_cap][P]
    float *stat = nullptr, *out = nullptr, *td = nullptr, *lossbuf = nullptr;   // [G][parts_cap][4], [G][4], [G][td_cap][2]
    float *scal = nullptr;                                 // [G][3]: log_alpha, its Adam exp_avg, exp_avg_sq
    int32_t td_cap = 0, parts_cap = 0, max_ctas = 4 * num_sms();
    int64_t epoch = 0, adam_t = 0;
    uint64_t calls = 0;
    // lockstep replay ring (continuous actions)
    float *frames = nullptr, *r_act2 = nullptr, *r_rew = nullptr;
    uint8_t *r_done = nullptr;
    int64_t ring_frames = 0, head = 0, count = 0;
    bool frame0_valid = false;
};

static int sac_pack(uavrl_sac *s, int role, cudaStream_t st)
{
    const NetDev &n = role == 0 ? s->sh.actor : s->sh.critic;
    pack_image_kernel<<<dim3((n.P + 255) / 256, s->G), 256, 0, st>>>(n.P, s->p[role], role == 0 ? s->map_a : s->map_c, s->img[role],
                                                                     n.smem_w_floats);
    UAVRL_LAUNCHED();
    return 0;
}

static void sac_fill_args(uavrl_sac *s, SacArgs &a, const BatchSrc &src, int B, const float *eps, uint64_t ctr)
{
    memset(&a, 0, sizeof(a));
    a.actor = s->sh.actor; a.critic = s->sh.critic; a.src = src; a.B = B; a.n_tiles = (B + kTile - 1) / kTile; a.gld = s->sh.gld;
    a.img_actor = s->img[0]; a.img_c1 = s->img[1]; a.img_c2 = s->img[2]; a.img_t1 = s->img[3]; a.img_t2 = s->img[4];
    a.eps = eps; a.key = s->cfg.seed ^ kNoiseSalt; a.ctr = ctr; a.log_alpha = s->scal; a.td = s->td;
    a.part_a = s->part[0]; a.part_c1 = s->part[1]; a.part_c2 = s->part[2]; a.stat = s->stat;
    a.h = SacHyper{ s->cfg.actor_lr, s->cfg.critic_lr, s->cfg.alpha_lr, s->cfg.target_entropy, s->cfg.gamma, s->cfg.tau, s->cfg.action_bound };
}

static void adam_args(AdamArgs &a, const NetDev &n, int nparts, float lr, int64_t t)
{
    memset(&a, 0, sizeof(a));
    a.P = n.P; a.nparts = nparts; a.n_loss_parts = 0; a.apply = 1; a.world = 1; a.img_floats = n.smem_w_floats;
    const double b1 = 0.9, b2 = 0.999;
    const double bc1 = 1.0 - pow(b1, (double)t), bc2 = 1.0 - pow(b2, (double)t);
    a.step_size = (float)((double)lr / bc1);
    a.beta1_c = (float)(1.0 - b1); a.beta2 = (float)b2; a.beta2_c = (float)(1.0 - b2);
    a.eps = 1e-8f; a.bc2_sqrt = (float)sqrt(bc2); a.inv_b = 1.f;
}

// gradient partial / stat slots per trainer for a per-trainer batch B: the tile kernels' grid.  They grow (never shrink) when a
// larger explicit batch arrives; TD targets likewise
static int sac_scratch(uavrl_sac *s, int B, int grid, cudaStream_t st)
{
    const size_t G = (size_t)s->G;
    int rc;
    if (grid > s->parts_cap) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        for (int r = 0; r < 3; ++r) { cudaFree(s->part[r]); s->part[r] = nullptr; }
        cudaFree(s->stat); s->stat = nullptr;
        s->parts_cap = 0;
        for (int r = 0; r < 3; ++r)
            if ((rc = dev_alloc(&s->part[r], G * grid * (size_t)(r == 0 ? s->sh.actor.P : s->sh.critic.P)))) return rc;
        if ((rc = dev_alloc(&s->stat, G * grid * 4))) return rc;
        s->parts_cap = grid;
    }
    if (B > s->td_cap) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        cudaFree(s->td); s->td = nullptr;
        s->td_cap = 0;
        if ((rc = dev_alloc(&s->td, G * B * kSacA))) return rc;
        s->td_cap = B;
    }
    return 0;
}

// one SAC_Trainer.update of every trainer on the batch described by src (B rows per trainer)
static int sac_update_impl(uavrl_sac *s, const BatchSrc &src, int B, const float *eps_next, const float *eps_cur, float *losses_dev, cudaStream_t st)
{
    const int n_tiles = (B + kTile - 1) / kTile;
    const int grid = n_tiles < s->max_ctas ? n_tiles : s->max_ctas;
    int rc = sac_scratch(s, B, grid, st);
    if (rc) return rc;
    const dim3 tiles(grid, s->G);                        // y: trainer
    SacArgs a;
    s->adam_t += 1;
    sac_fill_args(s, a, src, B, eps_next, 2 * (uint64_t)s->epoch);
    if (s->G > 1) sac_target_kernel<true><<<tiles, kNetThreads, smem_target(s->sh), st>>>(a);
    else sac_target_kernel<false><<<grid, kNetThreads, smem_target(s->sh), st>>>(a);
    UAVRL_LAUNCHED();
    if (s->G > 1) sac_critic_kernel<true><<<tiles, kNetThreads, smem_critic(s->sh), st>>>(a);
    else sac_critic_kernel<false><<<grid, kNetThreads, smem_critic(s->sh), st>>>(a);
    UAVRL_LAUNCHED();
    AdamArgs aa;
    for (int c = 1; c <= 2; ++c) {
        adam_args(aa, s->sh.critic, grid, s->cfg.critic_lr, s->adam_t);
        reduce_adam_kernel<<<dim3((aa.P + 63) / 64, s->G), 256, 0, st>>>(aa, s->part[c], s->lossbuf, s->grad[c], s->p[c], s->m[c], s->v[c], nullptr,
                                                                        s->img[c], nullptr, s->map_c, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                                        nullptr, nullptr);
        UAVRL_LAUNCHED();
    }
    sac_fill_args(s, a, src, B, eps_cur, 2 * (uint64_t)s->epoch + 1);
    if (s->G > 1) sac_actor_kernel<true><<<tiles, kNetThreads, smem_actor(s->sh), st>>>(a);
    else sac_actor_kernel<false><<<grid, kNetThreads, smem_actor(s->sh), st>>>(a);
    UAVRL_LAUNCHED();
    adam_args(aa, s->sh.actor, grid, s->cfg.actor_lr, s->adam_t);
    reduce_adam_kernel<<<dim3((aa.P + 63) / 64, s->G), 256, 0, st>>>(aa, s->part[0], s->lossbuf, s->grad[0], s->p[0], s->m[0], s->v[0], nullptr,
                                                                    s->img[0], nullptr, s->map_a, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                                    nullptr);
    UAVRL_LAUNCHED();
    SacFinishArgs f;
    memset(&f, 0, sizeof(f));
    f.Pc = s->sh.critic.P; f.nparts = grid; f.img_floats = s->sh.critic.smem_w_floats;
    f.tau = s->cfg.tau; f.alpha_lr = s->cfg.alpha_lr; f.target_entropy = s->cfg.target_entropy;
    f.inv_n = 1.f / ((float)B * (float)kSacA); f.do_alpha = 1;
    const double bc1 = 1.0 - pow(0.9, (double)s->adam_t), bc2 = 1.0 - pow(0.999, (double)s->adam_t);
    f.step_size_scale = (float)((double)s->cfg.alpha_lr / bc1); f.bc2_sqrt = (float)sqrt(bc2);
    sac_finish_kernel<<<dim3((f.Pc + 255) / 256, s->G), 256, 0, st>>>(f, s->stat, s->scal, s->p[1], s->p[2], s->p[3], s->p[4], s->img[3],
                                                                     s->img[4], s->map_c, losses_dev ? losses_dev : s->out);
    UAVRL_LAUNCHED();
    return 0;
}


// everything a learner allocates; on failure the caller destroys the half-built handle
static int sac_alloc(uavrl_sac *s)
{
    const uavrl_sac_config *cfg = &s->cfg;
    const size_t G = (size_t)s->G;
    int rc;
    for (int r = 0; r < 5; ++r) {
        const NetDev &n = r == 0 ? s->sh.actor : s->sh.critic;
        if ((rc = dev_alloc(&s->p[r], G * n.P)) || (rc = dev_alloc(&s->img[r], G * n.smem_w_floats))) return rc;
    }
    for (int r = 0; r < 3; ++r) {
        const NetDev &n = r == 0 ? s->sh.actor : s->sh.critic;
        if ((rc = dev_alloc(&s->m[r], G * n.P)) || (rc = dev_alloc(&s->v[r], G * n.P)) || (rc = dev_alloc(&s->grad[r], G * n.P))) return rc;
    }
    std::vector<int32_t> ma, mc;
    build_image_map(s->sh.actor, ma); build_image_map(s->sh.critic, mc);
    if ((rc = dev_alloc(&s->map_a, ma.size())) || (rc = dev_alloc(&s->map_c, mc.size()))) return rc;
    UAVRL_CUDA(cudaMemcpy(s->map_a, ma.data(), ma.size() * 4, cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(s->map_c, mc.data(), mc.size() * 4, cudaMemcpyHostToDevice));
    {   // gradient partial / stat slots per trainer: one learner keeps max_ctas (any batch); a grouped learner sizes them from the
        // per-trainer batch and grows them for larger explicit batches (sac_scratch)
        const int tiles = (cfg->batch_size + kTile - 1) / kTile;
        const int cap = (G == 1 || tiles > s->max_ctas) ? s->max_ctas : tiles;
        if ((rc = sac_scratch(s, cfg->batch_size, cap, 0))) return rc;
    }
    if ((rc = dev_alloc(&s->scal, 3 * G)) || (rc = dev_alloc(&s->out, 4 * G)) || (rc = dev_alloc(&s->lossbuf, 1))) return rc;
    std::vector<float> init(3 * G, 0.f);
    for (size_t g = 0; g < G; ++g) init[3 * g] = logf(0.01f);          // SAC_Trainer.py:53
    UAVRL_CUDA(cudaMemcpy(s->scal, init.data(), init.size() * 4, cudaMemcpyHostToDevice));
    if (cfg->lockstep_envs > 0) {
        // the ring holds, for every trainer, the frames a stand-alone learner with replay_capacity / G transitions over N / G
        // envs would keep
        const int64_t N = cfg->lockstep_envs, Ng = N / s->G, cap_g = cfg->replay_capacity / s->G;
        int64_t cap_frames = (cap_g + Ng - 1) / Ng;
        if (cap_frames < 2) cap_frames = 2;
        s->ring_frames = cap_frames + 1;
        const size_t slots = (size_t)s->ring_frames * N;
        if ((rc = dev_alloc(&s->frames, slots * cfg->obs_dim)) || (rc = dev_alloc(&s->r_act2, slots * kSacA)) || (rc = dev_alloc(&s->r_rew, slots)) ||
            (rc = dev_alloc(&s->r_done, slots)))
            return rc;
    }
    if ((rc = raise_dyn_smem(sac_target_kernel<false>, smem_target(s->sh))) || (rc = raise_dyn_smem(sac_critic_kernel<false>, smem_critic(s->sh))) ||
        (rc = raise_dyn_smem(sac_actor_kernel<false>, smem_actor(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<false>, smem_act(s->sh))) ||
        (rc = raise_dyn_smem(sac_target_kernel<true>, smem_target(s->sh))) || (rc = raise_dyn_smem(sac_critic_kernel<true>, smem_critic(s->sh))) ||
        (rc = raise_dyn_smem(sac_actor_kernel<true>, smem_actor(s->sh))) || (rc = raise_dyn_smem(sac_act_kernel<true>, smem_act(s->sh))))
        return rc;
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
    size_t b[4];
    if ((rc = sac_smem_total(sh, b))) return rc;
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
    if (n_trainers < 1 || n_trainers > 65535)        // every grouped kernel runs one grid row per trainer: gridDim.y <= 65535
        return fail(UAVRL_ERR_INVALID, "n_trainers must be in [1, 65535]");
    if (n_trainers > 1 && (cfg->lockstep_envs < 0 || cfg->lockstep_envs % n_trainers != 0))
        return fail(UAVRL_ERR_INVALID, "lockstep_envs must be a multiple of n_trainers (every trainer owns lockstep_envs / n_trainers envs)");
    if (n_trainers > 1 && cfg->replay_capacity / n_trainers <= 0)
        return fail(UAVRL_ERR_INVALID, "replay_capacity / n_trainers must be > 0");
    if (cfg->batch_size <= 0 || cfg->replay_capacity <= 0) return fail(UAVRL_ERR_INVALID, "batch_size and replay_capacity must be > 0");
    SacShape sh;
    int rc = sac_shape(*cfg, sh);
    if (rc) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(UAVRL_ERR_CUDA, "no CUDA device: the SAC learner has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg->device));
    size_t smem[4];
    if ((rc = sac_smem_total(sh, smem))) return rc;
    for (int i = 0; i < 4; ++i)
        if (smem[i] > kSacMaxSmem)
            return fail(UAVRL_ERR_INVALID, "networks too large for the SMEM-resident SAC kernels: " + std::to_string(smem[i]) +
                                               " B of shared memory per block, at most " + std::to_string(kSacMaxSmem));
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
        cudaGetLastError();                                  // a failed cudaMalloc must not surface at the next launch check
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
    for (int r = 0; r < 5; ++r) { cudaFree(s->p[r]); cudaFree(s->img[r]); }
    for (int r = 0; r < 3; ++r) { cudaFree(s->m[r]); cudaFree(s->v[r]); cudaFree(s->grad[r]); cudaFree(s->part[r]); }
    void *ptrs[] = { s->map_a, s->map_c, s->stat, s->scal, s->out, s->td, s->lossbuf, s->frames, s->r_act2, s->r_rew, s->r_done };
    for (void *p : ptrs) cudaFree(p);
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
    if (n % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_act: n must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    SacArgs a;
    BatchSrc none;
    memset(&none, 0, sizeof(none));
    const int ng = n / s->G;                                   // rows per trainer: block g belongs to trainer g
    sac_fill_args(s, a, none, ng, eps_dev, 0x8000000000000000ull | s->calls++);
    const int grid = a.n_tiles < s->max_ctas ? a.n_tiles : s->max_ctas;
    if (s->G > 1) sac_act_kernel<true><<<dim3(grid, s->G), kNetThreads, smem_act(s->sh), (cudaStream_t)stream>>>(a, obs_dev, ng, actions_dev);
    else sac_act_kernel<false><<<grid, kNetThreads, smem_act(s->sh), (cudaStream_t)stream>>>(a, obs_dev, ng, actions_dev);
    UAVRL_LAUNCHED();
    return 0;
}

int uavrl_sac_update_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                           const float *d_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev, void *stream)
{
    if (!s || B <= 0 || !s_dev || !a_dev || !r_dev || !s2_dev || !d_dev) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (B % s->G != 0) return fail(UAVRL_ERR_INVALID, "uavrl_sac_update_batch: B must be a multiple of the trainer count");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kBatchExplicit; src.frames = s_dev; src.s2_rows = s2_dev; src.act2 = a_dev; src.rew = r_dev; src.done_f32 = d_dev;
    return sac_update_impl(s, src, B / s->G, eps_next_dev, eps_cur_dev, losses_dev, (cudaStream_t)stream);
}

// the lockstep ring as a batch source: idx_tape (device, [G][batch_size] trainer-local logical indices, 0 = oldest) or Philox
// sampling keyed by the epoch.  Every trainer samples its own block of N / G envs (trainer_src), count = its transitions
static BatchSrc sac_ring_source(const uavrl_sac *s, const int32_t *idx_tape)
{
    const int64_t N = s->cfg.lockstep_envs, R = s->ring_frames;
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kReplayLockstep; src.frames = s->frames; src.act2 = s->r_act2; src.rew = s->r_rew; src.done_u8 = s->r_done;
    src.count = s->count / s->G; src.cap = R; src.n_envs = (int32_t)(N / s->G); src.row_stride = (int32_t)N;
    src.oldest = ((s->head - s->count / N) % R + R) % R;
    src.key = s->cfg.seed ^ kSampleSalt; src.epoch = (uint64_t)s->epoch;
    src.idx_tape = idx_tape;
    return src;
}

int64_t uavrl_sac_replay_size(const uavrl_sac *s) { return s ? s->count : 0; }

int uavrl_sac_replay_gather(uavrl_sac *s, int32_t n, const int64_t *idx, float *s_host, float *a_host, float *r_host, float *s2_host,
                            uint8_t *d_host)
{
    if (!s || n <= 0 || !idx) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (!s->frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    for (int i = 0; i < n; ++i)
        if (idx[i] < 0 || idx[i] >= s->count) return fail(UAVRL_ERR_INVALID, "logical index out of range");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    BatchSrc src = sac_ring_source(s, nullptr);
    src.n_envs = src.row_stride;                                // whole-ring logical indices, whatever the trainer count
    const size_t in = (size_t)s->cfg.obs_dim;
    int64_t *d_idx = nullptr; float *d_s = nullptr, *d_s2 = nullptr, *d_a = nullptr, *d_r = nullptr; uint8_t *d_d = nullptr;
    struct Free { void **p[6]; ~Free() { for (auto q : p) if (*q) cudaFree(*q); } } guard{ { (void **)&d_idx, (void **)&d_s, (void **)&d_s2,
                                                                                             (void **)&d_a, (void **)&d_r, (void **)&d_d } };
    UAVRL_CUDA(cudaMalloc((void **)&d_idx, (size_t)n * 8));
    UAVRL_CUDA(cudaMemcpy(d_idx, idx, (size_t)n * 8, cudaMemcpyHostToDevice));
    if (s_host) UAVRL_CUDA(cudaMalloc((void **)&d_s, (size_t)n * in * 4));
    if (s2_host) UAVRL_CUDA(cudaMalloc((void **)&d_s2, (size_t)n * in * 4));
    if (a_host) UAVRL_CUDA(cudaMalloc((void **)&d_a, (size_t)n * kSacA * 4));
    if (r_host) UAVRL_CUDA(cudaMalloc((void **)&d_r, (size_t)n * 4));
    if (d_host) UAVRL_CUDA(cudaMalloc((void **)&d_d, (size_t)n));
    sac_gather_kernel<<<(n + 7) / 8, 256>>>(n, (int)in, src, d_idx, d_s, d_s2, d_a, d_r, d_d);
    UAVRL_CUDA(cudaGetLastError());
    if (s_host) UAVRL_CUDA(cudaMemcpy(s_host, d_s, (size_t)n * in * 4, cudaMemcpyDeviceToHost));
    if (s2_host) UAVRL_CUDA(cudaMemcpy(s2_host, d_s2, (size_t)n * in * 4, cudaMemcpyDeviceToHost));
    if (a_host) UAVRL_CUDA(cudaMemcpy(a_host, d_a, (size_t)n * kSacA * 4, cudaMemcpyDeviceToHost));
    if (r_host) UAVRL_CUDA(cudaMemcpy(r_host, d_r, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (d_host) UAVRL_CUDA(cudaMemcpy(d_host, d_d, (size_t)n, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_sac_update_replay(uavrl_sac *s, const int32_t *idx_tape_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev,
                            void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    if (!s->frames) return fail(UAVRL_ERR_STATE, "the SAC learner has no replay ring (lockstep_envs == 0)");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    if (s->count / s->G <= s->cfg.batch_size) return 0;        // PathPlan_City.py:383: nothing sampled yet (per trainer)
    return sac_update_impl(s, sac_ring_source(s, idx_tape_dev), s->cfg.batch_size, eps_next_dev, eps_cur_dev, losses_dev, (cudaStream_t)stream);
}

int uavrl_sac_federate_actors(uavrl_sac *s, void *stream)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int P = s->sh.actor.P;
    sac_federate_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, s->G, s->p[0]);
    UAVRL_LAUNCHED();
    return sac_pack(s, 0, st);                                 // the G actor images
}

// lockstep loop with the continuous env step: state -> actor sample -> Move_Agent -> replay add -> update
int uavrl_sac_train_run(uavrl_env *env, uavrl_sac *s, int32_t n_iters, int32_t do_update, uavrl_train_stats *stats_host, void *stream)
{
    if (!env || !s || n_iters < 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (s->cfg.lockstep_envs != env->d.n || !s->frames) return fail(UAVRL_ERR_INVALID, "sac.lockstep_envs must equal env.n_envs");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_sac_train_run before uavrl_env_reset");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t N = env->d.n, in = s->cfg.obs_dim, R = s->ring_frames;
    unsigned long long c0[8] = { 0 }; double r0 = 0.0;
    if (stats_host) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        UAVRL_CUDA(cudaMemcpy(c0, env->d.stat_counts, sizeof(c0), cudaMemcpyDeviceToHost));
        UAVRL_CUDA(cudaMemcpy(&r0, env->d.stat_reward, sizeof(r0), cudaMemcpyDeviceToHost));
    }
    int rc; int64_t updates = 0;
    for (int it = 0; it < n_iters; ++it) {
        const int64_t f = s->head, fn = (s->head + 1) % R;
        float *obs_t = s->frames + f * N * in, *obs_next = s->frames + fn * N * in, *act = s->r_act2 + f * N * kSacA, *rew = s->r_rew + f * N;
        uint8_t *done = s->r_done + f * N;
        if (!s->frame0_valid) { if ((rc = launch_env_observe(env->d, obs_t, st))) return rc; s->frame0_valid = true; }
        if ((rc = uavrl_sac_act(s, obs_t, (int32_t)N, nullptr, act, st))) return rc;
        if ((rc = launch_env_step(env->d, UAVRL_ACT_CONT_F32X2, act, obs_next, rew, done, nullptr, nullptr, nullptr, st))) return rc;
        s->head = fn;
        const int64_t maxc = (R - 1) * N;
        s->count = s->count + N > maxc ? maxc : s->count + N;
        if (do_update) {
            s->epoch += 1;
            if (s->count / s->G <= s->cfg.batch_size) continue;     // per trainer
            if ((rc = sac_update_impl(s, sac_ring_source(s, nullptr), s->cfg.batch_size, nullptr, nullptr, nullptr, st))) return rc;
            ++updates;
        }
    }
    if (stats_host) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        unsigned long long c1[8]; double r1;
        UAVRL_CUDA(cudaMemcpy(c1, env->d.stat_counts, sizeof(c1), cudaMemcpyDeviceToHost));
        UAVRL_CUDA(cudaMemcpy(&r1, env->d.stat_reward, sizeof(r1), cudaMemcpyDeviceToHost));
        std::vector<float> o((size_t)s->G * 4);                 // [G][4]; last_loss = the mean actor loss over trainers
        UAVRL_CUDA(cudaMemcpy(o.data(), s->out, o.size() * sizeof(float), cudaMemcpyDeviceToHost));
        double lsum = 0.0;
        for (int g = 0; g < s->G; ++g) lsum += o[4 * (size_t)g];
        stats_host->env_steps = (int64_t)(c1[0] - c0[0]); stats_host->episodes_ended = (int64_t)(c1[1] - c0[1]);
        stats_host->collisions = (int64_t)(c1[2] - c0[2]); stats_host->n_success = (int64_t)(c1[3] - c0[3]);
        stats_host->n_lose = (int64_t)(c1[4] - c0[4]); stats_host->sum_reward = r1 - r0; stats_host->updates = updates;
        stats_host->last_loss = (float)(lsum / (double)s->G);
    }
    return 0;
}

}  // extern "C"
