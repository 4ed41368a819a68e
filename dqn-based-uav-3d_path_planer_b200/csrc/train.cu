// train.cu -- the fused lockstep training loop over the env batch and the learner.
//
// Replaces PathPlan_City.run_thread_OffPolicy + PathPlan_City.update (Envs/PathPlan_City.py:364-385,
// 757-776) for N envs: state -> get_action -> Move_Agent -> replay add -> sample -> Trainer.update.
// Observations are produced once by the env kernel, directly into the replay frame ring: the
// frame written as "next_obs" of iteration t is the "obs" the policy reads at t+1 (no copy, no
// separate push kernel; 412 B per stored transition instead of 812 B).
#include "env.cuh"
#include "learner.cuh"

#include <vector>

using namespace uavrl;

// the start of every lockstep iteration: begin the ring's iteration (the very first one also materialises obs_0), then
// Choose_Action2 -> Trainer.get_action (PathPlan_City.py:338-346) and Move_Agent + replay add (:371-382) -- reward/done land
// in the ring slots -- and commit the frame
static int act_step_commit(uavrl_env *env, uavrl_learner *l, float eps, cudaStream_t st)
{
    int rc;
    const ReplayStore::Iteration io = l->replay.begin();
    if (!l->replay.frame0_valid) {
        if ((rc = launch_env_observe(env->d, io.obs_t, st))) return rc;
        l->replay.frame0_valid = true;
    }
    if ((rc = launch_act(l, io.obs_t, env->d.n, eps, l->is_train, nullptr, nullptr, io.act, nullptr, st))) return rc;
    if ((rc = launch_env_step(env->d, UAVRL_ACT_DISCRETE27, io.act, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st,
                              l->pdl_prev == kPdlAct && g_pdl.load()))) return rc;
    l->pdl_prev = kPdlEnv;
    lockstep_commit(l, st);
    return 0;
}

extern "C" int uavrl_train_run(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t updates_per_iter,
                               int32_t do_update, uavrl_train_stats *stats_host, void *stream)
{
    if (!env || !l || n_iters < 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (l->replay.mode != kReplayLockstep || l->cfg.lockstep_envs != env->d.n)
        return fail(UAVRL_ERR_INVALID, "learner.lockstep_envs must equal env.n_envs");
    if (l->net.in_dim != kObsDim) return fail(UAVRL_ERR_INVALID, "learner.in_dim must be 100 (the UAV observation)");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_train_run before uavrl_env_reset");
    if (env->cfg.device != l->cfg.device) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    EnvStatsMark mark;
    if ((rc = mark.begin(env->d, st, stats_host))) return rc;
    int64_t updates = 0;
    l->pdl_chain = true; l->pdl_prev = kPdlNone;          // the first kernel of the loop is launched plainly
    struct ChainOff { uavrl_learner *l; ~ChainOff() { l->pdl_chain = false; l->pdl_prev = kPdlNone; } } chain_off{ l };
    for (int it = 0; it < n_iters; ++it) {
        if ((rc = act_step_commit(env, l, eps, st))) return rc;
        if (do_update) {
            for (int u = 0; u < updates_per_iter; ++u) {  // PathPlan_City.update -> Trainer.update (:757-776)
                l->epoch += 1;
                if (l->replay.count / l->G <= l->cfg.batch_size) continue;   // per trainer
                BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, nullptr);
                if ((rc = launch_update(l, src, l->cfg.batch_size, l->cfg.batch_size, l->loss_dev, true, st))) return rc;
                ++updates;
            }
        }
    }
    if ((rc = mark.end(env->d, st, updates, stats_host))) return rc;
    if (stats_host) {
        std::vector<float> losses((size_t)l->G);                // grouped learner: the mean over trainers
        UAVRL_CUDA(cudaMemcpy(losses.data(), l->loss_dev, losses.size() * sizeof(float), cudaMemcpyDeviceToHost));
        double lsum = 0.0;
        for (float x : losses) lsum += x;
        stats_host->last_loss = (float)(lsum / (double)l->G);
    }
    return 0;
}

extern "C" int uavrl_train_run_dp(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t global_batch, void *stream)
{
    if (!env || !l || n_iters < 0 || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (l->G > 1) return fail(UAVRL_ERR_INVALID, "uavrl_train_run_dp is not available on a learner with several trainers");
    if (l->replay.mode != kReplayLockstep || l->cfg.lockstep_envs != env->d.n)
        return fail(UAVRL_ERR_INVALID, "learner.lockstep_envs must equal env.n_envs");
    if (l->net.in_dim != kObsDim) return fail(UAVRL_ERR_INVALID, "learner.in_dim must be 100 (the UAV observation)");
    if (!l->comm_ready) return fail(UAVRL_ERR_STATE, "uavrl_train_run_dp before uavrl_learner_comm_connect");
    if (!env->reset_done) return fail(UAVRL_ERR_STATE, "uavrl_train_run_dp before uavrl_env_reset");
    if (env->cfg.device != l->cfg.device) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    // every rank must take part in every all-reduce, so every iteration must update: the caller warms the replay up first.
    // The count never shrinks, so the first iteration's sample decides, and a refusal leaves env, ring and epoch untouched
    if (n_iters > 0 && l->replay.count_after_commit() <= l->cfg.batch_size)
        return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions (warm up with uavrl_train_run first)");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    l->pdl_chain = true; l->pdl_prev = kPdlNone;
    struct ChainOff { uavrl_learner *l; ~ChainOff() { l->pdl_chain = false; l->pdl_prev = kPdlNone; } } chain_off{ l };
    for (int it = 0; it < n_iters; ++it) {
        if ((rc = act_step_commit(env, l, eps, st))) return rc;
        l->epoch += 1;
        BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, nullptr);
        if ((rc = launch_update_dp(l, src, l->cfg.batch_size, global_batch, l->loss_dev, st))) return rc;
    }
    return 0;
}

extern "C" int uavrl_train_profile(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, float *ms_out, void *stream)
{
    if (!env || !l || n_iters <= 0 || !ms_out) return fail(UAVRL_ERR_INVALID, "bad argument");
    if (l->net.in_dim != kObsDim) return fail(UAVRL_ERR_INVALID, "learner.in_dim must be 100 (the UAV observation)");
    if (env->cfg.device != l->cfg.device) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    if (l->replay.mode != kReplayLockstep || l->cfg.lockstep_envs != env->d.n || !env->reset_done || !l->replay.frame0_valid)
        return fail(UAVRL_ERR_STATE, "uavrl_train_profile needs a warmed-up lockstep env/learner pair");
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int NE = 7;                      // events per iteration -> 6 intervals
    std::vector<cudaEvent_t> ev((size_t)n_iters * NE);
    for (auto &e : ev) UAVRL_CUDA(cudaEventCreate(&e));
    int rc;
    for (int it = 0; it < n_iters; ++it) {
        const ReplayStore::Iteration io = l->replay.begin();
        cudaEvent_t *e = &ev[(size_t)it * NE];
        UAVRL_CUDA(cudaEventRecord(e[0], st));
        if ((rc = launch_act(l, io.obs_t, env->d.n, eps, l->is_train, nullptr, nullptr, io.act, nullptr, st))) return rc;
        UAVRL_CUDA(cudaEventRecord(e[1], st));
        if ((rc = launch_env_step(env->d, UAVRL_ACT_DISCRETE27, io.act, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st))) return rc;
        UAVRL_CUDA(cudaEventRecord(e[2], st));
        lockstep_commit(l, st);
        l->epoch += 1;
        if (l->replay.count / l->G <= l->cfg.batch_size) return fail(UAVRL_ERR_STATE, "replay not warmed up");
        BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, nullptr);
        if ((rc = launch_update_split(l, src, l->cfg.batch_size, st, &e[3]))) return rc;   // records e[3], e[4], e[5]
        UAVRL_CUDA(cudaEventRecord(e[6], st));
    }
    UAVRL_CUDA(cudaStreamSynchronize(st));
    for (int k = 0; k < NE - 1; ++k) ms_out[k] = 0.f;
    for (int it = 0; it < n_iters; ++it)
        for (int k = 0; k < NE - 1; ++k) {
            float ms = 0.f;
            UAVRL_CUDA(cudaEventElapsedTime(&ms, ev[(size_t)it * NE + k], ev[(size_t)it * NE + k + 1]));
            ms_out[k] += ms;
        }
    for (auto &e : ev) cudaEventDestroy(e);
    return 0;
}
