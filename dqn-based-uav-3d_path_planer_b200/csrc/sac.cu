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
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "env.cuh"
#include "mlp_tile.cuh"

namespace uavrl {

constexpr int kSacA = 2;                 // action_dim of the reference's UAV task (config/Trainer.xml:8,21)
constexpr int kGld = 64;                 // row stride of the gradient ping-pong planes

struct SacHyper { float actor_lr, critic_lr, alpha_lr, target_entropy, gamma, tau, bound; };

struct SacArgs {
    NetDev actor, critic;
    BatchSrc src;
    int32_t B, n_tiles;
    const float *img_actor, *img_c1, *img_c2, *img_t1, *img_t2;
    const float *eps;                    // [B][A] injected noise (nullptr -> Philox Box-Muller)
    uint64_t key, ctr;
    const float *log_alpha;              // device scalar
    float *td;                           // [B][A]
    float *part_a, *part_c1, *part_c2;   // gradient partials [grid][P]
    float *stat;                         // [grid][4]: critic-1 sq-err sum, critic-2 sq-err sum, actor-loss sum, entropy sum
    SacHyper h;
};

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ void noise2(const SacArgs &a, int gb, float &e0, float &e1)
{
    if (a.eps) { e0 = a.eps[2 * gb]; e1 = a.eps[2 * gb + 1]; return; }
    uint32_t r[4];
    Philox::gen(a.key, a.ctr, (uint64_t)gb, r);
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

// backward of one critic for the tile: dY (head gradient plane, [32][kGld], zero beyond the 2 outputs) -> optional parameter
// gradients into gpart, optional action-input gradient dA[32][A].  Planes of the critic live at rc + act_off.
__device__ void critic_backward_tile(const NetDev &cn, const float *sw, const float *rc, float *dY, float *dX, float *gpart,
                                     bool accumulate, float (*dA)[kSacA], int obs_dim)
{
    for (int l = cn.n_layers - 1; l >= 0; --l) {
        const LayerDev &L = cn.L[l];
        const float *Xin = rc + cn.act_off[l];
        const int ldx = cn.act_ld[l];
        if (gpart) layer_backward_dw(dY, kGld, Xin, ldx, gpart, L, accumulate);
        if (l > 0) {
            layer_backward_dx(dY, kGld, sw + L.smem_w, Xin, ldx, dX, kGld, L.in, L.out);
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
                for (int o = 0; o < L.out; ++o) s += dY[b * kGld + o] * w[o];
                dA[b][j] = s;
            }
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------ TD target (calc_target, :122-131)
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
    if (threadIdx.x == 0) { stage_weights(an, a.img_actor, RA, &bar[0]); stage_weights(cn, a.img_t1, RT1, &bar[1]); stage_weights(cn, a.img_t2, WT2, &bar[2]); }
    uint32_t pkey[4];
    Philox::gen(a.src.key, a.src.epoch, 0x5A17ull, pkey);
    const float alpha = expf(*a.log_alpha);
    bool ready = false;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s2 = nullptr; tr.r = 0.f; tr.d = 0.f;
            if (gb < a.B) tr = resolve_transition(a.src, gb, an.in_dim, pkey);
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
            if (gb < a.B) noise2(a, gb, e[0], e[1]);
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
                    a.td[(size_t)gb * kSacA + j] = s_r[b] + a.h.gamma * nv * (1.f - s_d[b]);
                }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ critic update (:343-360)
__global__ void __launch_bounds__(kNetThreads) sac_critic_kernel(SacArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &cn = a.critic;
    float *RC = smem, *WC2 = RC + cn.smem_total_floats;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * kGld, *Q = dYb + kTile * kGld;
    __shared__ uint64_t bar[2];
    __shared__ const float *rows[kTile];
    __shared__ float s_act[kTile][kSacA], s_sq[kTile];
    if (threadIdx.x == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) { stage_weights(cn, a.img_c1, RC, &bar[0]); stage_weights(cn, a.img_c2, WC2, &bar[1]); }
    uint32_t pkey[4];
    Philox::gen(a.src.key, a.src.epoch, 0x5A17ull, pkey);
    const float inv = 1.f / ((float)a.B * (float)kSacA);
    float sq[2] = { 0.f, 0.f };
    bool ready = false;
    int iter = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr; tr.ax = tr.ay = 0.f;
            if (gb < a.B) tr = resolve_transition(a.src, gb, cn.in_dim - kSacA, pkey);
            rows[threadIdx.x] = (gb < a.B) ? tr.s : nullptr; s_act[threadIdx.x][0] = tr.ax; s_act[threadIdx.x][1] = tr.ay;
        }
        __syncthreads();
        load_rows(rows, dYa, kGld * 2, cn.in_dim - kSacA);                  // stage s in the (still unused) gradient planes: 32 x 128
        __syncthreads();
        build_critic_input(dYa, kGld * 2, cn.in_dim - kSacA, RC + cn.act_off[0], cn.act_ld[0], s_act);
        if (!ready) { mbar_wait(&bar[0], 0); mbar_wait(&bar[1], 0); ready = true; }
        __syncthreads();
        for (int which = 0; which < 2; ++which) {
            const float *sw = which ? WC2 : RC;
            net_forward(cn, sw, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, Q);
            if (threadIdx.x < kTile) {
                const int b = threadIdx.x, gb = t * kTile + b;
                float *g = dYa + b * kGld;
                for (int o = 0; o < 32; ++o) g[o] = 0.f;
                float e2 = 0.f;
                if (gb < a.B)
                    for (int j = 0; j < kSacA; ++j) {
                        const float diff = Q[b * 32 + j] - a.td[(size_t)gb * kSacA + j];
                        e2 += diff * diff;
                        g[j] = 2.f * diff * inv;
                    }
                s_sq[b] = e2;
            }
            __syncthreads();
            if (threadIdx.x == 0) { float s = 0.f; for (int b = 0; b < kTile; ++b) s += s_sq[b]; sq[which] += s; }
            critic_backward_tile(cn, sw, RC, dYa, dYb, (which ? a.part_c2 : a.part_c1) + (size_t)blockIdx.x * cn.P, iter > 0, nullptr, 0);
        }
    }
    if (threadIdx.x == 0) { a.stat[blockIdx.x * 4 + 0] = sq[0]; a.stat[blockIdx.x * 4 + 1] = sq[1]; }
}

// ------------------------------------------------------------------ actor update (:362-376)
__global__ void __launch_bounds__(kNetThreads) sac_actor_kernel(SacArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor, &cn = a.critic;
    float *RA = smem, *RC = RA + an.smem_total_floats, *WC2 = RC + cn.smem_total_floats;
    float *dYa = WC2 + cn.smem_w_floats, *dYb = dYa + kTile * kGld, *head = dYb + kTile * kGld, *q1 = head + kTile * 32, *q2 = q1 + kTile * 32;
    __shared__ uint64_t bar[3];
    __shared__ const float *rows[kTile];
    __shared__ ActorOut s_o[kTile][kSacA];
    __shared__ float s_eps[kTile][kSacA], s_act[kTile][kSacA], s_dq1[kTile][kSacA], s_dq2[kTile][kSacA], s_dA1[kTile][kSacA],
        s_dA2[kTile][kSacA], s_l[kTile], s_e[kTile];
    if (threadIdx.x == 0) { for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) { stage_weights(an, a.img_actor, RA, &bar[0]); stage_weights(cn, a.img_c1, RC, &bar[1]); stage_weights(cn, a.img_c2, WC2, &bar[2]); }
    uint32_t pkey[4];
    Philox::gen(a.src.key, a.src.epoch, 0x5A17ull, pkey);
    const float alpha = expf(*a.log_alpha);
    const float inv = 1.f / ((float)a.B * (float)kSacA);
    float loss_acc = 0.f, ent_acc = 0.f;
    bool ready = false;
    int iter = 0;
    float *gpart = a.part_a + (size_t)blockIdx.x * an.P;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++iter) {
        if (threadIdx.x < kTile) {
            const int gb = t * kTile + threadIdx.x;
            Transition tr; tr.s = nullptr;
            if (gb < a.B) tr = resolve_transition(a.src, gb, an.in_dim, pkey);
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
            if (gb < a.B) noise2(a, gb, e[0], e[1]);
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
            float *g = dYa + b * kGld;
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
        critic_backward_tile(cn, WC2, RC, dYa, dYb, nullptr, false, s_dA2, an.in_dim);              // d/d a through critic 2
        net_forward(cn, RC, RC + cn.act_off[0], cn.act_ld[0], RC, true, nullptr, nullptr, q1);      // planes back to critic 1
        if (threadIdx.x < kTile) {
            float *g = dYa + threadIdx.x * kGld;
            for (int o = 0; o < 32; ++o) g[o] = 0.f;
            for (int j = 0; j < kSacA; ++j) g[j] = s_dq1[threadIdx.x][j];
        }
        __syncthreads();
        critic_backward_tile(cn, RC, RC, dYa, dYb, nullptr, false, s_dA1, an.in_dim);               // d/d a through critic 1
        // through tanh squash, reparameterisation, tanh / softplus heads to the head pre-activations
        if (threadIdx.x < kTile) {
            const int b = threadIdx.x;
            float *g = dYa + b * kGld;
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
            layer_backward_dw(dYa, kGld, RA + an.act_off[1], an.act_ld[1], gpart, L1, iter > 0);
            layer_backward_dx(dYa, kGld, RA + L1.smem_w, RA + an.act_off[1], an.act_ld[1], dYb, kGld, L1.in, L1.out);
            __syncthreads();
            layer_backward_dw(dYb, kGld, RA + an.act_off[0], an.act_ld[0], gpart, L0, iter > 0);
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) { a.stat[blockIdx.x * 4 + 2] = loss_acc; a.stat[blockIdx.x * 4 + 3] = ent_acc; }
}

// ------------------------------------------------------------------ alpha step + soft target update + scalar outputs
struct SacFinishArgs {
    int Pc, nparts;
    float tau, alpha_lr, target_entropy, inv_n, step_size_scale, bc2_sqrt;
    int do_alpha;
};

__global__ void sac_finish_kernel(SacFinishArgs f, const float *__restrict__ stat, float *__restrict__ scal, const float *__restrict__ c1,
                                  const float *__restrict__ c2, float *__restrict__ t1, float *__restrict__ t2, float *__restrict__ img_t1,
                                  float *__restrict__ img_t2, const int32_t *__restrict__ cmap, float *__restrict__ out)
{
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

// get_action (:444-448): action = actor(state)[0] with fresh noise
__global__ void __launch_bounds__(kNetThreads) sac_act_kernel(SacArgs a, const float *__restrict__ obs, int n, float *__restrict__ actions)
{
    extern __shared__ __align__(16) float smem[];
    const NetDev &an = a.actor;
    float *RA = smem, *head = RA + an.smem_total_floats;
    __shared__ uint64_t bar;
    __shared__ const float *rows[kTile];
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) stage_weights(an, a.img_actor, RA, &bar);
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
                noise2(a, gb, e[0], e[1]);
                for (int j = 0; j < kSacA; ++j) actions[(size_t)gb * kSacA + j] = actor_point(head[b * 32 + j], head[b * 32 + kSacA + j], e[j]).a * a.h.bound;
            }
        }
        __syncthreads();
    }
}

}  // namespace uavrl

using namespace uavrl;

// ------------------------------------------------------------------ host handle
struct uavrl_sac {
    uavrl_sac_config cfg;
    NetDev actor, critic;
    float *p[5] = { nullptr }, *img[5] = { nullptr };      // actor, c1, c2, t1, t2
    float *m[3] = { nullptr }, *v[3] = { nullptr }, *grad[3] = { nullptr };
    int32_t *map_a = nullptr, *map_c = nullptr;
    float *part[3] = { nullptr };                          // gradient partials
    float *stat = nullptr, *scal = nullptr, *out = nullptr, *td = nullptr, *lossbuf = nullptr;
    int32_t td_cap = 0, max_ctas = 4 * num_sms();
    int64_t epoch = 0, adam_t = 0;
    uint64_t calls = 0;
    // lockstep replay ring (continuous actions)
    float *frames = nullptr, *r_act2 = nullptr, *r_rew = nullptr;
    uint8_t *r_done = nullptr;
    int64_t ring_frames = 0, head = 0, count = 0;
    bool frame0_valid = false;
};

static size_t smem_target(const uavrl_sac *s) { return (size_t)(s->actor.smem_total_floats + s->critic.smem_total_floats + s->critic.smem_w_floats + 3 * kTile * 32) * 4; }
static size_t smem_critic(const uavrl_sac *s) { return (size_t)(s->critic.smem_total_floats + s->critic.smem_w_floats + 2 * kTile * kGld + kTile * 32) * 4; }
static size_t smem_actor(const uavrl_sac *s) { return (size_t)(s->actor.smem_total_floats + s->critic.smem_total_floats + s->critic.smem_w_floats + 2 * kTile * kGld + 3 * kTile * 32) * 4; }
static size_t smem_act(const uavrl_sac *s) { return (size_t)(s->actor.smem_total_floats + kTile * 32) * 4; }

static int sac_pack(uavrl_sac *s, int role, cudaStream_t st)
{
    const NetDev &n = role == 0 ? s->actor : s->critic;
    pack_image_kernel<<<(n.P + 255) / 256, 256, 0, st>>>(n.P, s->p[role], role == 0 ? s->map_a : s->map_c, s->img[role], 0);
    UAVRL_LAUNCHED();
    return 0;
}

static void sac_fill_args(uavrl_sac *s, SacArgs &a, const BatchSrc &src, int B, const float *eps, uint64_t ctr)
{
    memset(&a, 0, sizeof(a));
    a.actor = s->actor; a.critic = s->critic; a.src = src; a.B = B; a.n_tiles = (B + kTile - 1) / kTile;
    a.img_actor = s->img[0]; a.img_c1 = s->img[1]; a.img_c2 = s->img[2]; a.img_t1 = s->img[3]; a.img_t2 = s->img[4];
    a.eps = eps; a.key = s->cfg.seed ^ 0x5AC5ull; a.ctr = ctr; a.log_alpha = s->scal; a.td = s->td;
    a.part_a = s->part[0]; a.part_c1 = s->part[1]; a.part_c2 = s->part[2]; a.stat = s->stat;
    a.h = SacHyper{ s->cfg.actor_lr, s->cfg.critic_lr, s->cfg.alpha_lr, s->cfg.target_entropy, s->cfg.gamma, s->cfg.tau, s->cfg.action_bound };
}

static void adam_args(AdamArgs &a, int P, int nparts, float lr, int64_t t)
{
    memset(&a, 0, sizeof(a));
    a.P = P; a.nparts = nparts; a.n_loss_parts = 0; a.apply = 1; a.world = 1;
    const double b1 = 0.9, b2 = 0.999;
    const double bc1 = 1.0 - pow(b1, (double)t), bc2 = 1.0 - pow(b2, (double)t);
    a.step_size = (float)((double)lr / bc1);
    a.beta1_c = (float)(1.0 - b1); a.beta2 = (float)b2; a.beta2_c = (float)(1.0 - b2);
    a.eps = 1e-8f; a.bc2_sqrt = (float)sqrt(bc2); a.inv_b = 1.f;
}

// one SAC_Trainer.update on the batch described by src
static int sac_update_impl(uavrl_sac *s, const BatchSrc &src, int B, const float *eps_next, const float *eps_cur, float *losses_dev, cudaStream_t st)
{
    if (B > s->td_cap) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        cudaFree(s->td);
        UAVRL_CUDA(cudaMalloc((void **)&s->td, (size_t)B * kSacA * 4));
        s->td_cap = B;
    }
    SacArgs a;
    const int n_tiles = (B + kTile - 1) / kTile;
    const int grid = n_tiles < s->max_ctas ? n_tiles : s->max_ctas;
    s->adam_t += 1;
    sac_fill_args(s, a, src, B, eps_next, 2 * (uint64_t)s->epoch);
    sac_target_kernel<<<grid, kNetThreads, smem_target(s), st>>>(a);
    UAVRL_LAUNCHED();
    sac_critic_kernel<<<grid, kNetThreads, smem_critic(s), st>>>(a);
    UAVRL_LAUNCHED();
    AdamArgs aa;
    for (int c = 1; c <= 2; ++c) {
        adam_args(aa, s->critic.P, grid, s->cfg.critic_lr, s->adam_t);
        reduce_adam_kernel<<<(aa.P + 63) / 64, 256, 0, st>>>(aa, s->part[c], s->lossbuf, s->grad[c], s->p[c], s->m[c], s->v[c], nullptr, s->img[c],
                                                             nullptr, s->map_c, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
        UAVRL_LAUNCHED();
    }
    sac_fill_args(s, a, src, B, eps_cur, 2 * (uint64_t)s->epoch + 1);
    sac_actor_kernel<<<grid, kNetThreads, smem_actor(s), st>>>(a);
    UAVRL_LAUNCHED();
    adam_args(aa, s->actor.P, grid, s->cfg.actor_lr, s->adam_t);
    reduce_adam_kernel<<<(aa.P + 63) / 64, 256, 0, st>>>(aa, s->part[0], s->lossbuf, s->grad[0], s->p[0], s->m[0], s->v[0], nullptr, s->img[0], nullptr,
                                                         s->map_a, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    UAVRL_LAUNCHED();
    SacFinishArgs f;
    memset(&f, 0, sizeof(f));
    f.Pc = s->critic.P; f.nparts = grid; f.tau = s->cfg.tau; f.alpha_lr = s->cfg.alpha_lr; f.target_entropy = s->cfg.target_entropy;
    f.inv_n = 1.f / ((float)B * (float)kSacA); f.do_alpha = 1;
    const double bc1 = 1.0 - pow(0.9, (double)s->adam_t), bc2 = 1.0 - pow(0.999, (double)s->adam_t);
    f.step_size_scale = (float)((double)s->cfg.alpha_lr / bc1); f.bc2_sqrt = (float)sqrt(bc2);
    sac_finish_kernel<<<(f.Pc + 255) / 256, 256, 0, st>>>(f, s->stat, s->scal, s->p[1], s->p[2], s->p[3], s->p[4], s->img[3], s->img[4], s->map_c,
                                                         losses_dev ? losses_dev : s->out);
    UAVRL_LAUNCHED();
    return 0;
}

extern "C" {

int uavrl_sac_create(const uavrl_sac_config *cfg, uavrl_sac **out)
{
    if (!cfg || !out) return fail(UAVRL_ERR_INVALID, "uavrl_sac_create: null argument");
    if (cfg->act_dim != kSacA) return fail(UAVRL_ERR_INVALID, "act_dim must be 2 (the reference's UAV task)");
    if (cfg->batch_size <= 0 || cfg->replay_capacity <= 0) return fail(UAVRL_ERR_INVALID, "batch_size and replay_capacity must be > 0");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(UAVRL_ERR_CUDA, "no CUDA device: the SAC learner has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg->device));
    uavrl_sac *s = new uavrl_sac();
    s->cfg = *cfg;
    {   // grid cap of the tile kernels: 4 CTAs per SM's worth of tiles, i.e. one tile per CTA up to batch 4 x SMs x 32.  (One CTA
        // per SM looping over its tiles would accumulate ONE partial, at the price of a read-modify-write of the global partial
        // per tile.)
        const char *ov = getenv("UAVRL_SAC_MAX_CTAS");            // tests: force the multi-tile (accumulating) path on a small batch
        if (ov && atoi(ov) > 0) s->max_ctas = atoi(ov);
    }
    int rc;
    const int32_t ha[1] = { cfg->hidden }, hc[2] = { cfg->hidden, cfg->hidden };
    if ((rc = build_mlp(cfg->obs_dim, 1, ha, kSacA, kSacA, s->actor))) return rc;              // fc1 -> {fc_mu ; fc_std}
    if ((rc = build_mlp(cfg->obs_dim + kSacA, 2, hc, kSacA, 0, s->critic))) return rc;          // fc1 -> fc2 -> fc_out
    if (cfg->obs_dim % 4 != 0) return fail(UAVRL_ERR_INVALID, "obs_dim must be a multiple of 4");
    if (smem_target(s) > 227 * 1024 || smem_actor(s) > 227 * 1024) return fail(UAVRL_ERR_INVALID, "networks too large for the SMEM-resident SAC kernels");
    for (int r = 0; r < 5; ++r) {
        const NetDev &n = r == 0 ? s->actor : s->critic;
        if ((rc = dev_alloc(&s->p[r], (size_t)n.P)) || (rc = dev_alloc(&s->img[r], (size_t)n.smem_w_floats))) return rc;
    }
    for (int r = 0; r < 3; ++r) {
        const NetDev &n = r == 0 ? s->actor : s->critic;
        if ((rc = dev_alloc(&s->m[r], (size_t)n.P)) || (rc = dev_alloc(&s->v[r], (size_t)n.P)) || (rc = dev_alloc(&s->grad[r], (size_t)n.P)) ||
            (rc = dev_alloc(&s->part[r], (size_t)n.P * s->max_ctas)))
            return rc;
    }
    std::vector<int32_t> ma, mc;
    build_image_map(s->actor, ma); build_image_map(s->critic, mc);
    if ((rc = dev_alloc(&s->map_a, ma.size())) || (rc = dev_alloc(&s->map_c, mc.size()))) return rc;
    UAVRL_CUDA(cudaMemcpy(s->map_a, ma.data(), ma.size() * 4, cudaMemcpyHostToDevice));
    UAVRL_CUDA(cudaMemcpy(s->map_c, mc.data(), mc.size() * 4, cudaMemcpyHostToDevice));
    if ((rc = dev_alloc(&s->stat, (size_t)4 * s->max_ctas)) || (rc = dev_alloc(&s->scal, 4)) || (rc = dev_alloc(&s->out, 4)) ||
        (rc = dev_alloc(&s->lossbuf, (size_t)s->max_ctas)) || (rc = dev_alloc(&s->td, (size_t)cfg->batch_size * kSacA)))
        return rc;
    s->td_cap = cfg->batch_size;
    const float la0 = logf(0.01f);                                     // SAC_Trainer.py:53
    UAVRL_CUDA(cudaMemcpy(s->scal, &la0, 4, cudaMemcpyHostToDevice));
    if (cfg->lockstep_envs > 0) {
        const int64_t N = cfg->lockstep_envs;
        int64_t cap_frames = (cfg->replay_capacity + N - 1) / N;
        if (cap_frames < 2) cap_frames = 2;
        s->ring_frames = cap_frames + 1;
        const size_t slots = (size_t)s->ring_frames * N;
        if ((rc = dev_alloc(&s->frames, slots * cfg->obs_dim)) || (rc = dev_alloc(&s->r_act2, slots * kSacA)) || (rc = dev_alloc(&s->r_rew, slots)) ||
            (rc = dev_alloc(&s->r_done, slots)))
            return rc;
    }
    UAVRL_CUDA(cudaFuncSetAttribute(sac_target_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_target(s)));
    UAVRL_CUDA(cudaFuncSetAttribute(sac_critic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_critic(s)));
    UAVRL_CUDA(cudaFuncSetAttribute(sac_actor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_actor(s)));
    UAVRL_CUDA(cudaFuncSetAttribute(sac_act_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_act(s)));
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

int64_t uavrl_sac_param_count(const uavrl_sac *s, int32_t role) { return !s ? 0 : (role == 0 ? s->actor.P : s->critic.P); }

static float *sac_buf(uavrl_sac *s, int role)
{
    if (role >= 0 && role < 5) return s->p[role];
    if (role >= 5 && role < 8) return s->m[role - 5];
    if (role >= 8 && role < 11) return s->v[role - 8];
    return nullptr;
}

int uavrl_sac_set_params(uavrl_sac *s, int32_t role, const float *h)
{
    if (!s || !h || !sac_buf(s, role)) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const int rr = role < 5 ? role : (role - 5) % 3;
    const int P = rr == 0 ? s->actor.P : s->critic.P;
    UAVRL_CUDA(cudaMemcpy(sac_buf(s, role), h, (size_t)P * 4, cudaMemcpyHostToDevice));
    if (role < 5) { int rc = sac_pack(s, role, 0); if (rc) return rc; UAVRL_CUDA(cudaDeviceSynchronize()); }
    return 0;
}

int uavrl_sac_get_params(uavrl_sac *s, int32_t role, float *h)
{
    if (!s || !h || !sac_buf(s, role)) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const int rr = role < 5 ? role : (role - 5) % 3;
    const int P = rr == 0 ? s->actor.P : s->critic.P;
    UAVRL_CUDA(cudaMemcpy(h, sac_buf(s, role), (size_t)P * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int uavrl_sac_set_scalars(uavrl_sac *s, float log_alpha, float la_m, float la_v, int64_t epoch, int64_t adam_step)
{
    if (!s) return fail(UAVRL_ERR_INVALID, "null handle");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    UAVRL_CUDA(cudaDeviceSynchronize());
    const float v[3] = { log_alpha, la_m, la_v };
    UAVRL_CUDA(cudaMemcpy(s->scal, v, sizeof(v), cudaMemcpyHostToDevice));
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
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    SacArgs a;
    BatchSrc none;
    memset(&none, 0, sizeof(none));
    sac_fill_args(s, a, none, n, eps_dev, 0x8000000000000000ull | s->calls++);
    const int grid = a.n_tiles < s->max_ctas ? a.n_tiles : s->max_ctas;
    sac_act_kernel<<<grid, kNetThreads, smem_act(s), (cudaStream_t)stream>>>(a, obs_dev, n, actions_dev);
    UAVRL_LAUNCHED();
    return 0;
}

int uavrl_sac_update_batch(uavrl_sac *s, int32_t B, const float *s_dev, const float *a_dev, const float *r_dev, const float *s2_dev,
                           const float *d_dev, const float *eps_next_dev, const float *eps_cur_dev, float *losses_dev, void *stream)
{
    if (!s || B <= 0 || !s_dev || !a_dev || !r_dev || !s2_dev || !d_dev) return fail(UAVRL_ERR_INVALID, "bad argument");
    UAVRL_CUDA(cudaSetDevice(s->cfg.device));
    s->epoch += 1;                                             // SAC_Trainer.py:320
    BatchSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = kBatchExplicit; src.frames = s_dev; src.s2_rows = s2_dev; src.act2 = a_dev; src.rew = r_dev; src.done_f32 = d_dev;
    return sac_update_impl(s, src, B, eps_next_dev, eps_cur_dev, losses_dev, (cudaStream_t)stream);
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
            if (s->count <= s->cfg.batch_size) continue;
            BatchSrc src;
            memset(&src, 0, sizeof(src));
            src.mode = kReplayLockstep; src.frames = s->frames; src.act2 = s->r_act2; src.rew = s->r_rew; src.done_u8 = s->r_done;
            src.count = s->count; src.cap = R; src.n_envs = (int32_t)N;
            src.oldest = ((s->head - s->count / N) % R + R) % R;
            src.key = s->cfg.seed ^ 0x5EEDull; src.epoch = (uint64_t)s->epoch;
            if ((rc = sac_update_impl(s, src, s->cfg.batch_size, nullptr, nullptr, nullptr, st))) return rc;
            ++updates;
        }
    }
    if (stats_host) {
        UAVRL_CUDA(cudaStreamSynchronize(st));
        unsigned long long c1[8]; double r1; float o[4];
        UAVRL_CUDA(cudaMemcpy(c1, env->d.stat_counts, sizeof(c1), cudaMemcpyDeviceToHost));
        UAVRL_CUDA(cudaMemcpy(&r1, env->d.stat_reward, sizeof(r1), cudaMemcpyDeviceToHost));
        UAVRL_CUDA(cudaMemcpy(o, s->out, sizeof(o), cudaMemcpyDeviceToHost));
        stats_host->env_steps = (int64_t)(c1[0] - c0[0]); stats_host->episodes_ended = (int64_t)(c1[1] - c0[1]);
        stats_host->collisions = (int64_t)(c1[2] - c0[2]); stats_host->n_success = (int64_t)(c1[3] - c0[3]);
        stats_host->n_lose = (int64_t)(c1[4] - c0[4]); stats_host->sum_reward = r1 - r0; stats_host->updates = updates;
        stats_host->last_loss = o[0];
    }
    return 0;
}

}  // extern "C"
