// train.cu -- the fused lockstep training loops over the env batch and a learner: the Q-network learner's (uavrl_train_run,
// uavrl_train_run_dp, uavrl_train_profile) and the SAC learner's (uavrl_sac_train_run, uavrl_sac_train_run_dp) run the same
// iteration.
//
// Replaces PathPlan_City.run_thread_OffPolicy + PathPlan_City.update (Envs/PathPlan_City.py:364-385,
// 757-776) for N envs: state -> get_action -> Move_Agent -> replay add -> sample -> Trainer.update.
// Observations are produced once by the env kernel, directly into the replay frame ring: the
// frame written as "next_obs" of iteration t is the "obs" the policy reads at t+1 (no copy, no
// separate push kernel; 412 B per stored transition instead of 812 B).
#include "env.cuh"
#include "learner.cuh"
#include "sac.cuh"

#include <vector>

using namespace uavrl;

enum Loop { kLoopRun, kLoopDp, kLoopProfile };

// ------------------------------------------------------------------ what the loop does differently per learner
// uavrl_learner_comm_connect / uavrl_sac_comm_connect has run: the data-parallel loop's precondition
static bool connected(const uavrl_learner *l) { return l->comm.ready; }
static bool connected(const uavrl_sac *s) { return s->comm.ready; }
static const char *connect_fn(const uavrl_learner *) { return "uavrl_learner_comm_connect"; }
static const char *connect_fn(const uavrl_sac *) { return "uavrl_sac_comm_connect"; }

// get_action on the ring's current frame: Choose_Action2 -> Trainer.get_action (PathPlan_City.py:338-346)
static int act(uavrl_learner *l, const ReplayStore::Iteration &io, int n, float eps, cudaStream_t st)
{
    return launch_act(l, io.obs_t, n, eps, l->is_train, nullptr, nullptr, io.act, nullptr, st);
}
static int act(uavrl_sac *s, const ReplayStore::Iteration &io, int n, float, cudaStream_t st)
{
    if (s->cfg.discrete) return launch_sacd_act(s, io.obs_t, n, nullptr, io.act, st);
    return launch_sac_act(s, io.obs_t, n, nullptr, io.act2, st);
}

// Move_Agent + replay add (:371-382) on those actions: reward / done land in the ring slots, the observations in the next frame.
// The Q-network's step joins the learner's dependent-launch chain.
static int env_step(uavrl_env *env, uavrl_learner *l, const ReplayStore::Iteration &io, cudaStream_t st)
{
    if (int rc = launch_env_step(env, UAVRL_ACT_DISCRETE27, io.act, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st,
                                 l->chain.next(kChainEnv).pdl))
        return rc;
    l->chain.launched(kChainEnv);
    return 0;
}
static int env_step(uavrl_env *env, uavrl_sac *s, const ReplayStore::Iteration &io, cudaStream_t st)
{
    if (s->cfg.discrete) return launch_env_step(env, UAVRL_ACT_DISCRETE27, io.act, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st);
    return launch_env_step(env, UAVRL_ACT_CONT_F32X2, io.act2, io.obs_next, io.rew, io.done, nullptr, nullptr, nullptr, st);
}

// the commit's prioritised-replay priority fill launches outside the Q-network's dependent-launch chain
static void committed(uavrl_learner *l) { if (l->replay.per_enabled()) l->chain.launched(kChainNone); }
static void committed(uavrl_sac *) {}

// PathPlan_City.update -> Trainer.update (:757-776) on batch_size transitions per trainer sampled through src.  dp_batch > 0:
// data-parallel over that global batch; marks (profiling, may be null): launch_update's three events
static int update(uavrl_learner *l, const BatchSrc &src, int dp_batch, cudaStream_t st, cudaEvent_t *marks)
{
    const int B = l->cfg.batch_size;
    return dp_batch > 0 ? launch_update_dp(l, src, B, dp_batch, l->loss_dev, st) : launch_update(l, src, B, B, l->loss_dev, true, st, marks);
}
static int update(uavrl_sac *s, const BatchSrc &src, int dp_batch, cudaStream_t st, cudaEvent_t *)
{
    const int B = s->cfg.batch_size;
    return dp_batch > 0 ? launch_sac_update_dp(s, src, B, dp_batch, nullptr, nullptr, nullptr, st)
                        : launch_sac_update(s, src, B, nullptr, nullptr, nullptr, st);
}

// where each trainer's loss of its last update lives: element 0 of [G][stride] device floats
struct Losses { const float *dev; int stride; };
static Losses losses(const uavrl_learner *l) { return { l->loss_dev, 1 }; }
static Losses losses(const uavrl_sac *s) { return { s->out, 4 }; }       // actor, critic 1, critic 2, alpha loss

// the loop refusals of one learner kind; null: none
static const char *learner_refusal(const uavrl_learner *, Loop) { return nullptr; }
static const char *learner_refusal(const uavrl_sac *s, Loop loop)
{
    if (!s->cfg.discrete) return nullptr;
    if (loop == kLoopDp) return "uavrl_sac_train_run_dp is not available on a discrete SAC learner";
    return s->cfg.act_dim == 27 ? nullptr : "a discrete SAC learner in the loop must have act_dim 27 (the discrete-27 step)";
}

// ------------------------------------------------------------------ the loop
// The refusals the loops share, each loop's in the order it reports them; nothing is enqueued before they pass.  fn: the entry
// point, named in the reset refusal.
template <class Learner>
static int check_loop(const uavrl_env *env, const Learner *l, Loop loop, int32_t n_iters, const char *fn)
{
    const ReplayStore &rs = l->replay;
    const bool paired = rs.mode == kReplayLockstep && l->cfg.lockstep_envs == env->d.n;
    if (const char *why = learner_refusal(l, loop)) return fail(UAVRL_ERR_INVALID, why);
    if (loop == kLoopDp && l->G > 1) return fail(UAVRL_ERR_INVALID, std::string(fn) + " is not available on a learner with several trainers");
    if (loop != kLoopProfile && !paired) return fail(UAVRL_ERR_INVALID, "learner.lockstep_envs must equal env.n_envs");
    // the env step writes kObsDim floats per env into the ring's frames
    if (rs.in_dim != kObsDim) return fail(UAVRL_ERR_INVALID, "learner.in_dim must be 100 (the UAV observation)");
    if (loop == kLoopDp && !connected(l)) return fail(UAVRL_ERR_STATE, std::string(fn) + " before " + connect_fn(l));
    if (loop != kLoopProfile && !env->reset_done) return fail(UAVRL_ERR_STATE, std::string(fn) + " before uavrl_env_reset");
    if (env->cfg.device != l->cfg.device) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    if (loop == kLoopProfile && (!paired || !env->reset_done || !rs.frame0_valid))
        return fail(UAVRL_ERR_STATE, "uavrl_train_profile needs a warmed-up lockstep env/learner pair");
    // the data-parallel loop: every rank must take part in every all-reduce; the profile: every iteration's update is timed.
    // So every iteration must update: the caller warms the replay up first.  The count never shrinks, so the first
    // iteration's sample decides, and a refusal leaves env, ring and epoch untouched
    if (loop != kLoopRun && n_iters > 0 && !rs.ready_after_commit(l->cfg.batch_size))
        return fail(UAVRL_ERR_STATE, "replay holds <= batch_size transitions (warm up with uavrl_train_run first)");
    return 0;
}

// One lockstep iteration: begin the ring's iteration (the very first one also materialises obs_0), act, env step, commit the
// frame, then n_updates updates, each counting an epoch and skipped while a trainer's ring holds <= batch_size transitions.
// ev (profiling, may be null): 7 events, before act, after act, after the env step, the update's three marks
// (launch_update), after the optimiser step.
template <class Learner>
static int iteration(uavrl_env *env, Learner *l, float eps, int n_updates, int dp_batch, cudaStream_t st, cudaEvent_t *ev,
                     int64_t &updates)
{
    int rc;
    ReplayStore &rs = l->replay;
    const ReplayStore::Iteration io = rs.begin();
    if (!rs.frame0_valid) {
        if ((rc = launch_env_observe(env, io.obs_t, st))) return rc;
        rs.frame0_valid = true;
    }
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[0], st));
    if ((rc = act(l, io, env->d.n, eps, st))) return rc;
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[1], st));
    if ((rc = env_step(env, l, io, st))) return rc;
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[2], st));
    if ((rc = rs.commit(st))) return rc;
    committed(l);
    for (int u = 0; u < n_updates; ++u) {
        l->epoch += 1;
        if (!rs.ready(l->cfg.batch_size)) continue;
        if ((rc = update(l, rs.source(l->cfg.seed, l->epoch, nullptr), dp_batch, st, ev ? ev + 3 : nullptr))) return rc;
        ++updates;
    }
    if (ev) UAVRL_CUDA(cudaEventRecord(ev[6], st));
    return 0;
}

// n_iters iterations of n_updates updates each; stats_host (may be null) receives what they added
template <class Learner>
static int run(uavrl_env *env, Learner *l, const char *fn, int32_t n_iters, float eps, int n_updates, uavrl_train_stats *stats_host,
               void *stream)
{
    int rc;
    if ((rc = check_loop(env, l, kLoopRun, n_iters, fn))) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    cudaStream_t st = (cudaStream_t)stream;
    EnvStatsMark mark;
    if ((rc = mark.begin(env->d, st, stats_host))) return rc;
    int64_t updates = 0;
    for (int it = 0; it < n_iters; ++it)
        if ((rc = iteration(env, l, eps, n_updates, 0, st, nullptr, updates))) return rc;
    if ((rc = mark.end(env->d, st, updates, stats_host))) return rc;
    if (stats_host) {
        const Losses ls = losses(l);                            // grouped learner: the mean over trainers
        std::vector<float> v((size_t)l->G * ls.stride);
        UAVRL_CUDA(cudaMemcpy(v.data(), ls.dev, v.size() * sizeof(float), cudaMemcpyDeviceToHost));
        double lsum = 0.0;
        for (size_t g = 0; g < (size_t)l->G; ++g) lsum += v[g * ls.stride];
        stats_host->last_loss = (float)(lsum / (double)l->G);
    }
    return 0;
}

extern "C" int uavrl_train_run(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t updates_per_iter,
                               int32_t do_update, uavrl_train_stats *stats_host, void *stream)
{
    if (!env || !l || n_iters < 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    ChainScope chain(l->chain);
    return run(env, l, "uavrl_train_run", n_iters, eps, do_update ? updates_per_iter : 0, stats_host, stream);
}

extern "C" int uavrl_sac_train_run(uavrl_env *env, uavrl_sac *s, int32_t n_iters, int32_t do_update, uavrl_train_stats *stats_host,
                                   void *stream)
{
    if (!env || !s || n_iters < 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    return run(env, s, "uavrl_sac_train_run", n_iters, 0.f, do_update ? 1 : 0, stats_host, stream);
}

// n_iters iterations whose update is the data-parallel one over global_batch
template <class Learner>
static int run_dp(uavrl_env *env, Learner *l, const char *fn, int32_t n_iters, float eps, int32_t global_batch, void *stream)
{
    int rc;
    if ((rc = check_loop(env, l, kLoopDp, n_iters, fn))) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    int64_t updates = 0;
    for (int it = 0; it < n_iters; ++it)
        if ((rc = iteration(env, l, eps, 1, global_batch, (cudaStream_t)stream, nullptr, updates))) return rc;
    return 0;
}

extern "C" int uavrl_train_run_dp(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, int32_t global_batch, void *stream)
{
    if (!env || !l || n_iters < 0 || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    ChainScope chain(l->chain);
    return run_dp(env, l, "uavrl_train_run_dp", n_iters, eps, global_batch, stream);
}

extern "C" int uavrl_sac_train_run_dp(uavrl_env *env, uavrl_sac *s, int32_t n_iters, int32_t global_batch, void *stream)
{
    if (!env || !s || n_iters < 0 || global_batch <= 0) return fail(UAVRL_ERR_INVALID, "bad argument");
    return run_dp(env, s, "uavrl_sac_train_run_dp", n_iters, 0.f, global_batch, stream);
}

// the loop of uavrl_train_run with the chain off and an event between every two kernels
extern "C" int uavrl_train_profile(uavrl_env *env, uavrl_learner *l, int32_t n_iters, float eps, float *ms_out, void *stream)
{
    if (!env || !l || n_iters <= 0 || !ms_out) return fail(UAVRL_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = check_loop(env, l, kLoopProfile, n_iters, "uavrl_train_profile"))) return rc;
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
