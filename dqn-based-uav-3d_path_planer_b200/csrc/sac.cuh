// sac.cuh -- host handle of the SAC learner (sac.cu) and the launches the lockstep loop (train.cu) makes on it.
#pragma once
#include "replay.cuh"
#include "net.cuh"
#include "optim.cuh"

namespace uavrl {
// the two networks of a SAC learner and the stride of its gradient planes: everything the kernels' shared memory follows from
struct SacShape { NetDev actor, critic; int32_t gld; };
}  // namespace uavrl

// A grouped learner (uavrl_sac_create_trainers) holds G trainers: every per-network vector, weight image and scratch array
// below is [G][...]; trainer g acts for envs [g Ng, (g + 1) Ng) of the shared ring frames and samples only their transitions.
struct uavrl_sac {
    uavrl_sac_config cfg;
    uavrl::SacShape sh;
    int32_t G = 1;
    float *p[5] = { nullptr }, *img[5] = { nullptr };      // actor, c1, c2, t1, t2
    float *m[3] = { nullptr }, *v[3] = { nullptr }, *grad[3] = { nullptr };
    // the data-parallel exchange vectors, one per phase of an update: xc = [grad c1 | grad c2 | critic-1, critic-2 squared-error
    // sums], xa = [grad actor | actor-loss sum, entropy sum] (grad[r] point into them; with G > 1 the gradients are [G][P] and
    // only a one-trainer learner exchanges)
    float *xc = nullptr, *xa = nullptr;
    int32_t *map_a = nullptr, *map_c = nullptr;
    float *part[3] = { nullptr };                          // gradient partials [G][parts_cap][P]
    float *stat = nullptr, *out = nullptr, *td = nullptr, *lossbuf = nullptr;   // [G][parts_cap][4], [G][4], [G][td_cap][2]
    float *scal = nullptr;                                 // [G][3]: log_alpha, its Adam exp_avg, exp_avg_sq
    int32_t td_cap = 0, parts_cap = 0, max_ctas = 4 * uavrl::num_sms();
    int64_t epoch = 0, adam_t = 0;
    uint64_t calls = 0;
    uavrl::ReplayStore replay;                             // lockstep ring (float[2] actions); none when lockstep_envs == 0
    // data-parallel training: the fused exchange's buffers (slots of max(2 Pc + 2, Pa + 2) words), and the split form's
    // phase (0 none, 1 critic gradients written, 2 critics stepped, 3 actor gradients written) with the batch it runs on
    uavrl::PeerComm comm;
    int32_t dp_phase = 0, dp_B = 0, dp_global = 0;
    uavrl::BatchSrc dp_src;
    // sharded actor aggregation (uavrl_sac_fed_shard): the trainers are global trainers [fed_rank G, (fed_rank + 1) G) of
    // G fed_world; fed_x [G fed_world][Pa] holds every trainer's actor once gathered, fed_phase 1 once the own slice is written
    int32_t fed_rank = 0, fed_world = 0, fed_phase = 0;
    float *fed_x = nullptr;
    uavrl::DevMem mem, parts_mem, td_mem, fed_mem;         // owners: networks, moments, maps, scalars; partials / stat; td; fed_x
};

namespace uavrl {
// SAC_Trainer.get_action of every trainer: n rows in G equal blocks (block g -> trainer g), actions [n][2]; eps (may be null)
// [n][2] injects the reparameterisation noise, else Philox on the learner's act-call counter
int launch_sac_act(uavrl_sac *s, const float *obs, int n, const float *eps, float *actions, cudaStream_t st);
// the same pass for an evaluation (eval.cu): noise from counter ctr without advancing the act-call counter, or with mean the
// policy's mean action tanh(mu) bound
int launch_sac_act_eval(uavrl_sac *s, const float *obs, int n, bool mean, uint64_t ctr, float *actions, cudaStream_t st);
// one SAC_Trainer.update of every trainer on the batch described by src (B rows per trainer); losses_dev (may be null: the
// learner's own out) receives [G][4]
int launch_sac_update(uavrl_sac *s, const BatchSrc &src, int B, const float *eps_next, const float *eps_cur, float *losses_dev,
                      cudaStream_t st);
// the data-parallel form over global_batch rows (B on this rank): the critics' gradients and squared-error sums go through one
// fused exchange + Adam, then the actor's gradient, loss and entropy sums through a second; every rank ends bit-identical
int launch_sac_update_dp(uavrl_sac *s, const BatchSrc &src, int B, int global_batch, const float *eps_next, const float *eps_cur,
                         float *losses_dev, cudaStream_t st);
}  // namespace uavrl
