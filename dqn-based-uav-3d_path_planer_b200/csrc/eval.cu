// eval.cu -- policy evaluation on the device: episodes of a trained learner over a held-out scenario suite, one episode record
// each (uavrl_eval_run for the Q-network learner, uavrl_sac_eval_run for SAC).
//
// The reference leaves its evaluation hooks as stubs (PathPlan_City.Evaluation_Action / Sim) and only reports counts while it
// trains.  Here the suite is pool scenarios first + k (mod P), k in [0, n): env e plays suite positions e, N + e, 2N + e, ...
// -- the env's own auto-reset with stride N -- and parks once it has none left.  Each iteration is the lockstep loop's act and
// env step without the ring: observe once, then act -> step, the step writing the next observations in place.  The records
// ride on the env step (uavrl_env_set_records, env_block.cuh): slot j N + e of env e's j-th episode is its suite position.
#include "env.cuh"
#include "learner.cuh"
#include "sac.cuh"

#include <algorithm>

using namespace uavrl;

// The sampled SAC evaluation's noise counter: Philox key seed ^ kNoiseSalt as every SAC draw (trainer g: seed + g), on counters
// of their own -- bit 62 set (act calls set bit 63, the updates count epochs from 0), then first_scenario and the iteration
constexpr uint64_t kEvalNoiseTag = 0x4000000000000000ull;
constexpr int kEvalPollIters = 64;      // iterations between two reads of the device's record count

// ------------------------------------------------------------------ what differs per learner
static int trainers(const uavrl_learner *l) { return l->G; }
static int trainers(const uavrl_sac *s) { return s->G; }
static int device(const uavrl_learner *l) { return l->cfg.device; }
static int device(const uavrl_sac *s) { return s->cfg.device; }
static int obs_dim(const uavrl_learner *l) { return l->cfg.in_dim; }
static int obs_dim(const uavrl_sac *s) { return s->cfg.obs_dim; }
// the env step's action kind; null: the learner cannot drive it
static const char *action_refusal(const uavrl_learner *l, int) { return l->cfg.n_actions == 27 ? nullptr : "the learner must have 27 actions (the discrete-27 step)"; }
static const char *action_refusal(const uavrl_sac *, int mean) { return (mean == 0 || mean == 1) ? nullptr : "mean_action must be 0 or 1"; }

struct EvalBufs { DevMem mem; float *obs = nullptr, *act_f = nullptr; int32_t *act_i = nullptr; };

// Trainer.get_action with Is_Train = 0 (greedy, DuelingDQN_Trainer.py:90): not an act call, so its Philox counter stays
static int act_step(uavrl_env *env, uavrl_learner *l, EvalBufs &b, int, int, int64_t, cudaStream_t st)
{
    const int n = env->d.n;
    const uint64_t calls = l->act_calls;
    int rc = launch_act(l, b.obs, n, 0.f, 0, nullptr, nullptr, b.act_i, nullptr, st);
    l->act_calls = calls;
    if (rc) return rc;
    return launch_env_step(env, UAVRL_ACT_DISCRETE27, b.act_i, b.obs, nullptr, nullptr, nullptr, nullptr, nullptr, st);
}
// SAC_Trainer.get_action (:444-448) on the evaluation's own noise stream, or the mean action
static int act_step(uavrl_env *env, uavrl_sac *s, EvalBufs &b, int mean, int first, int64_t it, cudaStream_t st)
{
    const uint64_t ctr = kEvalNoiseTag | ((uint64_t)(uint32_t)first << 31) | ((uint64_t)it & 0x7fffffffull);
    if (int rc = launch_sac_act_eval(s, b.obs, env->d.n, mean != 0, ctr, b.act_f, st)) return rc;
    return launch_env_step(env, UAVRL_ACT_CONT_F32X2, b.act_f, b.obs, nullptr, nullptr, nullptr, nullptr, nullptr, st);
}

// Refusals, before anything is enqueued
template <class Learner>
static int check_eval(const uavrl_env *env, const Learner *l, int32_t n_episodes, int64_t max_iters, int mean)
{
    if (n_episodes < 0 || max_iters < 0) return fail(UAVRL_ERR_INVALID, "n_episodes and max_iters must be >= 0");
    if (!env->pool_set) return fail(UAVRL_ERR_STATE, "evaluation before uavrl_env_set_pool: the suite is drawn from the pool");
    if (obs_dim(l) != kObsDim) return fail(UAVRL_ERR_INVALID, "the learner's input must be 100 wide (the UAV observation)");
    if (env->cfg.device != device(l)) return fail(UAVRL_ERR_INVALID, "env and learner live on different devices");
    if (env->d.n % trainers(l) != 0) return fail(UAVRL_ERR_INVALID, "n_envs must be a multiple of the trainer count");
    if (const char *why = action_refusal(l, mean)) return fail(UAVRL_ERR_INVALID, why);
    return 0;
}

// What the call changes on the env besides its state, put back however it returns: the records, auto-reset and stride
struct EnvEvalScope {
    uavrl_env *env;
    EnvRecords saved;
    int32_t auto_reset, stride, extras;
    bool active = false;
    explicit EnvEvalScope(uavrl_env *e) : env(e), auto_reset(e->d.auto_reset), stride(e->d.reset_stride), extras(e->d.extras) {}
    int begin(int64_t n)
    {
        EnvRecords r;
        if (int rc = records_alloc(r, env->d.n, std::max<int64_t>(n, 1))) return rc;
        r.dev.limit = n;
        saved = std::move(env->records);
        env->records = std::move(r);
        env->d.extras |= kExtraRecord;
        env->d.auto_reset = 1;
        env->d.reset_stride = env->d.n;
        active = true;
        return 0;
    }
    ~EnvEvalScope()
    {
        if (!active) return;
        cudaDeviceSynchronize();                                // nothing may still write the records being swapped back
        env->records = std::move(saved);
        env->d.extras = extras; env->d.auto_reset = auto_reset; env->d.reset_stride = stride;
    }
};

template <class Learner>
static int eval_run(uavrl_env *env, Learner *l, int32_t first_scenario, int32_t n_episodes, int32_t mean, int64_t max_iters,
                    uavrl_episode_record *records_host, uavrl_eval_stats *stats_host, void *stream)
{
    if (int rc = check_eval(env, l, n_episodes, max_iters, mean)) return rc;
    UAVRL_CUDA(cudaSetDevice(env->cfg.device));
    uavrl_eval_stats stats = { 0, 0, 0 };
    if (n_episodes == 0) {
        if (stats_host) *stats_host = stats;
        return 0;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const int N = env->d.n;
    const int64_t n = n_episodes;
    const int first = (int)(((int64_t)first_scenario % env->d.P + env->d.P) % env->d.P);
    // every segment ends within max_step steps, so ceil(n / N) episodes of at most K segments each end within this bound
    const int64_t bound = max_iters > 0 ? max_iters : ((n + N - 1) / N) * (int64_t)env->d.K * env->d.k.max_step;
    EvalBufs b;
    int rc;
    if ((rc = b.mem.alloc(b.obs, (size_t)N * kObsDim, false)) || (rc = b.mem.alloc(b.act_i, (size_t)N, false)) ||
        (rc = b.mem.alloc(b.act_f, (size_t)N * 2, false)))
        return rc;
    EnvEvalScope scope(env);
    if ((rc = scope.begin(n))) return rc;
    if ((rc = launch_env_reset(env, first, (int)std::min<int64_t>(n, N), st))) return rc;
    if ((rc = launch_env_observe(env, b.obs, st))) return rc;
    unsigned long long counts[2] = { 0, 0 };
    int64_t it = 0;
    while (it < bound && (int64_t)counts[0] < n) {
        const int64_t end = std::min(bound, it + kEvalPollIters);
        for (; it < end; ++it)
            if ((rc = act_step(env, l, b, mean, first, it, st))) return rc;
        UAVRL_CUDA(cudaMemcpyAsync(counts, env->records.dev.counts, sizeof(counts), cudaMemcpyDeviceToHost, st));
        UAVRL_CUDA(cudaStreamSynchronize(st));
    }
    if (records_host) UAVRL_CUDA(cudaMemcpy(records_host, env->records.dev.rec, (size_t)n * sizeof(uavrl_episode_record), cudaMemcpyDeviceToHost));
    stats.iterations = it;
    stats.records = (int64_t)counts[0];
    stats.unfinished = n - (int64_t)counts[0];
    if (stats_host) *stats_host = stats;
    return 0;
}

extern "C" int uavrl_eval_run(uavrl_env *env, uavrl_learner *l, int32_t first_scenario, int32_t n_episodes, int64_t max_iters,
                              uavrl_episode_record *records_host, uavrl_eval_stats *stats_host, void *stream)
{
    if (!env || !l) return fail(UAVRL_ERR_INVALID, "bad argument");
    return eval_run(env, l, first_scenario, n_episodes, 0, max_iters, records_host, stats_host, stream);
}

extern "C" int uavrl_sac_eval_run(uavrl_env *env, uavrl_sac *s, int32_t first_scenario, int32_t n_episodes, int32_t mean_action,
                                  int64_t max_iters, uavrl_episode_record *records_host, uavrl_eval_stats *stats_host, void *stream)
{
    if (!env || !s) return fail(UAVRL_ERR_INVALID, "bad argument");
    return eval_run(env, s, first_scenario, n_episodes, mean_action, max_iters, records_host, stats_host, stream);
}
