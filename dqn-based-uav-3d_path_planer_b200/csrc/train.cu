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

enum Loop { kLoopRun, kLoopDp, kLoopProfile };

// The refusals the three loops share, each loop's in the order it reports them; nothing is enqueued before they pass.
static int check_loop(const uavrl_env *env, const uavrl_learner *l, Loop loop, int32_t n_iters)
{
    const bool paired = l->replay.mode == kReplayLockstep && l->cfg.lockstep_envs == env->d.n;
    if (loop == kLoopDp && l->G > 1) return fail(UAVRL_ERR_INVALID, "uavrl_train_run_dp is not available on a learner with several trainers");
    if (loop != kLoopProfile && !paired) return fail(UAVRL_ERR_INVALID, "learner.lockstep_envs must equal env.n_envs");
    if (l->net.in_dim != kObsDim) return fail(UAVRL_ERR_INVALID, "learner.in_dim must be 100 (the UAV observation)");
    if (loop == kLoopDp && !l->comm_ready) return fail(UAVRL_ERR_STATE, "uavrl_train_run_dp before uavrl_learner_comm_connect");
    if (loop != kLoopProfile && !env->reset_done)
        return fail(UAVRL_ERR_STATE, loop == kLoopDp ? "uavrl_train_run_dp before uavrl_env_reset" : "uavrl_train_run before uavrl_env_reset");
    if (env->cfg.device != l->cfg.device) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    if (loop == kLoopProfile && (!paired || !env->reset_done || !l->replay.frame0_valid))
        return fail(UAVRL_ERR_STATE, "uavrl_train_profile needs a warmed-up lockstep env/learner pair");
    // the data-parallel loop: every rank must take part in every all-reduce; the profile: every iteration's update is timed.
    // So every iteration must update: the caller warms the replay up first.  The count never shrinks, so the first
    // iteration's sample decides, and a refusal leaves env, ring and epoch untouched
    if (loop != kLoopRun && n_iters > 0 && l->replay.count_after_commit() / l->G <= l->cfg.batch_size)
        return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions (warm up with uavrl_train_run first)");
    return 0;
}

// One lockstep iteration: begin the ring's iteration (the very first one also materialises obs_0), Choose_Action2 ->
// Trainer.get_action (PathPlan_City.py:338-346) and Move_Agent + replay add (:371-382) -- reward/done land in the ring slots --
// commit the frame, then n_updates x PathPlan_City.update -> Trainer.update (:757-776), each counting an epoch and skipped
// while a trainer's ring holds <= batch_size transitions.  dp_batch > 0: data-parallel updates over that global batch.
// ev (profiling, may be null): 7 events, before act, after act, after the env step, the update's three marks
// (launch_update), after the optimiser step.
static int iteration(uavrl_env *env, uavrl_learner *l, float eps, int n_updates, int dp_batch, cudaStream_t st, cudaEvent_t *ev,
                     int64_t &updates)
{
    int rc;
    const ReplayStore::Iteration io = l->replay.begin();
    if (!l->replay.frame0_valid) {
        if ((rc = launch_env_observe(env->d, io.obs_t, st))) return rc;
        l->replay.frame0_valid = true;
    }
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[0], st));
    if ((rc = launch_act(l, io.obs_t, env->d.n, eps, l->is_train, nullptr, nullptr, io.act, nullptr, st))) return rc;
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[1], st));
    if ((rc = launch_env_step(env->d, UAVRL_ACT_DISCRETE27, io.act, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st,
                              l->chain.next(kChainEnv).pdl))) return rc;
    l->chain.launched(kChainEnv);
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[2], st));
    lockstep_commit(l, st);
    const int B = l->cfg.batch_size;
    for (int u = 0; u < n_updates; ++u) {
        l->epoch += 1;
        if (l->replay.count / l->G <= B) continue;      // per trainer
        const BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, nullptr);
        if ((rc = dp_batch > 0 ? launch_update_dp(l, src, B, dp_batch, l->loss_dev, st)
                               : launch_update(l, src, B, B, l->loss_dev, true, st, ev ? ev + 3 : nullptr))) return rc;
        ++updates;
    }
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[6], st));
    return 0;
}

extern "C" int uavrl_train_run(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t updates_per_iter,
                               int32_t do_update, uavrl_train_stats *stats_host, void *stream)
{
    if (!env || !l || n_iters < 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = check_loop(env, l, kLoopRun, n_iters))) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    EnvStatsMark mark;
    if ((rc = mark.begin(env->d, st, stats_host))) return rc;
    int64_t updates = 0;
    {
        ChainScope chain(l->chain);
        for (int it = 0; it < n_iters; ++it)
            if ((rc = iteration(env, l, eps, do_update ? updates_per_iter : 0, 0, st, nullptr, updates))) return rc;
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
    int rc;
    if ((rc = check_loop(env, l, kLoopDp, n_iters))) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    ChainScope chain(l->chain);
    int64_t updates = 0;
    for (int it = 0; it < n_iters; ++it)
        if ((rc = iteration(env, l, eps, 1, global_batch, (cudaStream_t)stream, nullptr, updates))) return rc;
    return 0;
}

// the loop of uavrl_train_run with the chain off and an event between every two kernels
extern "C" int uavrl_train_profile(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, float *ms_out, void *stream)
{
    if (!env || !l || n_iters <= 0 || !ms_out) return fail(UAVRL_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = check_loop(env, l, kLoopProfile, n_iters))) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int NE = 7;                      // events per iteration -> 6 intervals
    std::vector<cudaEvent_t> ev((size_t)n_iters * NE);
    for (auto &e : ev) UAVRL_CUDA(cudaEventCreate(&e));
    int64_t updates = 0;
    for (int it = 0; it < n_iters; ++it)
        if ((rc = iteration(env, l, eps, 1, 0, st, &ev[(size_t)it * NE], updates))) return rc;
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
