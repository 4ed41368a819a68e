// replay.cuh -- the replay store shared by the Q-network and SAC learners: its layouts, the device view a batch is sampled
// through, and the host handle that owns it.
//
// Two layouts:
//   paired    (lockstep_envs == 0): slot s holds the rows frames[2 s] (state) and frames[2 s + 1] (next state), written by
//             uavrl_replay_push; a FIFO over `slots` transitions.
//   lockstep  (lockstep_envs = N > 0): the frame ring frames[F + 1][N][in].  The env step writes observation t + 1 straight into
//             frame t + 1, so transition (f, e) is (frames[f][e], act, rew, frames[f + 1][e], done) and its slot is f N + e.
//             Trainer g of a grouped learner owns envs [g Ng, (g + 1) Ng); its k-th oldest transition is the ring's logical
//             index (k / Ng) N + g Ng + k mod Ng.
#pragma once
#include "common.cuh"
#include "per.cuh"

namespace uavrl {

enum ReplayMode { kReplayPaired = 0, kReplayLockstep = 1, kBatchExplicit = 2 };

// where the rows of a batch come from
struct BatchSrc {
    int32_t mode;
    const float *frames;              // replay observation rows [rows][in_dim]
    const int32_t *act;               // [slots] discrete action index (DQN family)
    const float *act2;                // [slots][2] continuous action (SAC); nullptr otherwise
    const float *rew;                 // [slots]
    const uint8_t *done_u8;           // [slots]  (replay)          } one of the two
    const float *done_f32;            // [B]      (explicit batch)  }
    const float *s2_rows;             // explicit: next-state rows [B][in]
    const int32_t *idx_tape;          // optional injected indices [B]: logical (k-th oldest), or physical slots if idx_is_slot
    int32_t idx_is_slot;
    const float *is_w;                // optional per-sample importance weights (prioritised replay): loss = mean(w (Q-y)^2)
    float *abs_err;                   // optional out: |Q - y| per sample (ReplayTree.batch_update input)
    int64_t count, oldest;            // valid transitions, logical index of the oldest
    int64_t cap;                      // paired: slots ; lockstep: frames in the ring
    int32_t n_envs;                   // lockstep only: envs one trainer samples (count = frames x n_envs)
    int32_t row_stride;               // lockstep only: envs per ring frame (0 = n_envs); > n_envs for a grouped learner
    int32_t env_base;                 // lockstep only: first env sampled (trainer_src sets g x n_envs)
    uint64_t key, epoch;              // Philox key / counter for sampling
};

// Philox key salts of a learner seeded with `seed`: the eps-greedy draws use seed ^ kActSalt, replay sampling seed ^ kSampleSalt.
// Trainer g of a grouped learner draws exactly what a stand-alone learner seeded with seed + g draws.
// Federation probe draws (federate.cu) use seed ^ kFedSalt.
// Prioritised-replay draws (per.cu) use seed ^ kPerSalt.
constexpr uint64_t kActSalt = 0xAC7ull, kSampleSalt = 0x5EEDull, kFedSalt = 0xFEDull, kPerSalt = 0x9E12ull;
__host__ __device__ __forceinline__ uint64_t trainer_key(uint64_t key, uint64_t salt, int g) { return ((key ^ salt) + (uint64_t)g) ^ salt; }

// Host and device: the host compile lets the sampler be checked without a GPU.
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}

// i-th element of a keyed pseudo-random permutation of [0, M): 4-round Feistel on 2*h bits with
// cycle walking.  perm(0..B-1) = B distinct uniform indices = random.sample(range(M), B)
// (BaseClass/replay_buffer.py:49).
__host__ __device__ __forceinline__ uint64_t perm_index(uint64_t i, uint64_t M, const uint32_t key[4])
{
    int bits = 1;
    while ((1ull << bits) < M) ++bits;
    const int h = (bits + 1) / 2;
    const uint32_t mask = (h >= 32) ? 0xffffffffu : ((1u << h) - 1u);
    uint64_t x = i;
    do {
        uint32_t Lh = (uint32_t)(x >> h) & mask, Rh = (uint32_t)x & mask;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const uint32_t f = mix32(Rh ^ key[r]) & mask;
            const uint32_t nl = Rh;
            Rh = Lh ^ f;
            Lh = nl;
        }
        x = ((uint64_t)Lh << h) | Rh;
    } while (x >= M);
    return x;
}

#if defined(__CUDACC__)
// Trainer g's view of a batch source (grouped learner: gridDim.y = G trainers, B rows each).  Explicit batches: block g of the
// G x B rows.  Lockstep ring: env block [g n_envs, (g + 1) n_envs), trainer g's sampling key and row g of a [G][B] index tape.
// Both: row g of [G][B] importance weights and |Q - y| outputs (prioritised replay).
__device__ __forceinline__ BatchSrc trainer_src(BatchSrc s, int g, int B, int in_dim)
{
    if (g == 0) return s;
    const size_t r0 = (size_t)g * (size_t)B;
    if (s.is_w) s.is_w += r0;
    if (s.abs_err) s.abs_err += r0;
    if (s.mode == kBatchExplicit) {
        s.frames += r0 * in_dim; s.s2_rows += r0 * in_dim; s.rew += r0; s.done_f32 += r0;
        if (s.act) s.act += r0;
        if (s.act2) s.act2 += 2 * r0;
        return s;
    }
    s.env_base = g * s.n_envs;
    s.key = trainer_key(s.key, kSampleSalt, g);
    if (s.idx_tape) s.idx_tape += r0;
    return s;
}

// A replay transition's place: its slot (action / reward / done) and the rows of its state and next state
struct ReplayRef { int64_t slot, row, row2; };

// The layout of both replay modes: logical index j (the j-th oldest of the source's view), or a physical slot when idx_is_slot.
// fresh (optional): the next-state row lies in the frame the env step of the SAME iteration writes (lockstep ring: the frame
// behind the newest transition group) -- the only sampled row a kernel launched programmatically behind that env step must not
// read early
__device__ __forceinline__ ReplayRef replay_ref(const BatchSrc &src, uint64_t j, bool *fresh = nullptr)
{
    ReplayRef r;
    if (src.mode == kReplayLockstep) {
        const int64_t N = src.row_stride ? src.row_stride : src.n_envs;
        const int64_t f = src.idx_is_slot ? (int64_t)(j / src.n_envs) : (src.oldest + (int64_t)(j / src.n_envs)) % src.cap;
        const int64_t e = src.env_base + (int64_t)(j % src.n_envs);
        r.slot = f * N + e; r.row = r.slot;
        r.row2 = ((f + 1) % src.cap) * N + e;
        if (fresh) *fresh = ((f + 1) % src.cap) == (src.oldest + src.count / src.n_envs) % src.cap;
    } else {
        r.slot = src.idx_is_slot ? (int64_t)j : (src.oldest + (int64_t)j) % src.cap; r.row = 2 * r.slot; r.row2 = 2 * r.slot + 1;
    }
    return r;
}

// batch position gb -> the replay transition it samples (an index tape entry, or the gb-th element of the keyed permutation)
__device__ __forceinline__ ReplayRef replay_pick(const BatchSrc &src, int gb, const uint32_t pkey[4], bool *fresh = nullptr)
{
    return replay_ref(src, src.idx_tape ? (uint64_t)src.idx_tape[gb] : perm_index((uint64_t)gb, (uint64_t)src.count, pkey), fresh);
}

// batch position gb -> the transition's state row, next-state row and metadata
struct Transition { const float *s, *s2; int a; float r, d, ax, ay; };
// the two halves of resolve_transition: (1) where the rows are -- index arithmetic only, nothing a predecessor kernel writes is
// read (an index tape, when present, comes from a kernel that is never a programmatic-launch predecessor); (2) the
// transition's action / reward / done, which the env step of the same iteration may just have written
__device__ __forceinline__ int64_t resolve_rows(const BatchSrc &src, int gb, int in_dim, const uint32_t pkey[4], const float *&s, const float *&s2,
                                                bool *fresh = nullptr)
{
    if (fresh) *fresh = false;
    if (src.mode == kBatchExplicit) {
        s = src.frames + (size_t)gb * in_dim; s2 = src.s2_rows + (size_t)gb * in_dim;
        return gb;
    }
    const ReplayRef r = replay_pick(src, gb, pkey, fresh);
    s = src.frames + (size_t)r.row * in_dim; s2 = src.frames + (size_t)r.row2 * in_dim;
    return r.slot;
}
__device__ __forceinline__ void load_meta(const BatchSrc &src, int64_t slot, int &a, float &r, float &d)
{
    a = src.act ? src.act[slot] : 0; r = src.rew[slot];
    d = (src.mode == kBatchExplicit) ? src.done_f32[slot] : (src.done_u8[slot] ? 1.f : 0.f);
}
__device__ __forceinline__ Transition resolve_transition(const BatchSrc &src, int gb, int in_dim, const uint32_t pkey[4])
{
    Transition t;
    if (src.mode == kBatchExplicit) {
        t.s = src.frames + (size_t)gb * in_dim;
        t.s2 = src.s2_rows + (size_t)gb * in_dim;
        t.a = src.act ? src.act[gb] : 0; t.r = src.rew[gb]; t.d = src.done_f32[gb];
        t.ax = src.act2 ? src.act2[2 * gb] : 0.f; t.ay = src.act2 ? src.act2[2 * gb + 1] : 0.f;
        return t;
    }
    const ReplayRef r = replay_pick(src, gb, pkey);
    const int64_t slot = r.slot;
    t.s = src.frames + (size_t)r.row * in_dim;
    t.s2 = src.frames + (size_t)r.row2 * in_dim;
    t.a = src.act ? src.act[slot] : 0; t.r = src.rew[slot]; t.d = src.done_u8[slot] ? 1.f : 0.f;
    t.ax = src.act2 ? src.act2[2 * slot] : 0.f; t.ay = src.act2 ? src.act2[2 * slot + 1] : 0.f;
    return t;
}
#endif

// The replay store of one learner (host handle of device arrays).  Actions are int32 indices (Q-network) or float[2]
// (SAC); exactly one of act / act2 is allocated.
struct ReplayStore {
    int32_t mode = kReplayPaired;
    int32_t N = 0, G = 1, in_dim = 0;     // envs per ring frame (lockstep), trainers sharing it, row width
    float *frames = nullptr;
    int32_t *act = nullptr;
    float *act2 = nullptr;
    float *rew = nullptr;
    uint8_t *done = nullptr;
    int64_t slots = 0;                // paired: capacity ; lockstep: ring_frames * N
    int64_t ring_frames = 0;          // lockstep: frames in the ring (= capacity frames + 1)
    int64_t head = 0;                 // paired: next slot to write ; lockstep: frame holding obs_t
    int64_t count = 0;                // valid transitions
    bool frame0_valid = false;        // lockstep: frame `head` holds the current observations
    DevMem mem;                       // owns frames, act / act2, rew and done
    PerTree per;                      // prioritised replay: one SumTree per trainer over its own slots (per.cuh)

    // capacity transitions over all trainers; N > 0: lockstep ring, where every trainer keeps the frames a stand-alone store
    // with capacity / G transitions over N / G envs would keep (at least 2); N == 0: paired rows
    int alloc(int64_t capacity, int32_t n_envs, int32_t n_trainers, int32_t in, bool pair_actions);
    // trainer-local sampling: Philox keyed by seed ^ kSampleSalt and the epoch, or a device tape of logical indices
    BatchSrc source(uint64_t seed, int64_t epoch, const int32_t *idx_tape) const;
    // paired rows: n transitions at head (the oldest are overwritten once full), with prioritised replay at the priority of an
    // error-less push
    int push(int32_t n, const float *obs, const int32_t *a, const float *r, const float *next_obs, const uint8_t *d, cudaStream_t st);
    // lockstep iteration: where this iteration's observations, actions, rewards and done flags go; commit makes them a
    // transition group (the oldest is dropped once the ring is full), with prioritised replay first giving that group the
    // priority of an error-less push and the dropped one 0
    struct Iteration { float *obs_t, *obs_next; int32_t *act; float *act2, *rew; uint8_t *done; };
    Iteration begin() const;
    int commit(cudaStream_t st);
    int64_t count_after_commit() const;   // lockstep: `count` once the next commit has run
    // an update of `batch` transitions per trainer may sample (PathPlan_City.py:383): every trainer holds more than batch, now or
    // (lockstep) once the next commit has run
    bool ready(int64_t batch) const { return count / G > batch; }
    bool ready_after_commit(int64_t batch) const { return count_after_commit() / G > batch; }
    // forget every transition and clear the trees; the next iteration re-observes into frame `head`
    int restart();
    // n whole-store logical indices (0 = oldest) to host arrays; any output may be null
    int gather(int32_t n, const int64_t *idx, float *s, int32_t *a, float *a2, float *r, float *s2, uint8_t *d) const;

    // ---- prioritised replay (per.cu).  Every call acts on each trainer's tree at once (grid y = G) under trainer-local slots.
    bool per_enabled() const { return per.dev.enabled != 0; }
    // G trees of slots / G leaves; a negative hyper-parameter takes the reference's default.  Refused once a transition is
    // stored, and on a grouped paired store
    int per_enable(double alpha, double beta0, double beta_inc, double eps, double err_upper);
    // contiguous slots (mod cap) of every tree: the first n_first get `value`, the rest `value_rest` (n_first < 0: all get `value`)
    int per_fill_range(int64_t first_slot, int64_t n, double value, cudaStream_t st, int64_t n_first = -1, double value_rest = 0.0);
    // [G][n] slots: explicit priorities (prio), or the push (clip = 0) / batch_update (clip = 1) rule on |errors|
    int per_set(int n, const int32_t *slot_in, const double *prio, const float *abs_err, int clip, cudaStream_t st);
    // ReplayTree.sample2 of B per trainer, keyed by seed ^ kPerSalt: [G][B] slots and weights (null: the scratch per.dev.idx /
    // per.dev.w), uniforms from u_tape [G][B] when given
    int per_sample(uint64_t seed, int B, const double *u_tape, int32_t *slot_out, float *w_out, cudaStream_t st);
    // host read-back after a device synchronise: leaves [G][cap], totals [G], beta; any output may be null
    int per_get(double *leaves, double *total, double *beta) const;
    // every tree's leaves and sums to 0 (beta and the sampling counter are kept)
    int per_clear();
    // an update samples through the trees when they are enabled, the batch comes from the store and no index tape is injected
    bool per_samples(const BatchSrc &src) const { return per_enabled() && src.mode != kBatchExplicit && !src.idx_tape; }
    // such an update's batch: ReplayTree.sample2 of B per trainer into the scratch, and src reading its rows, importance
    // weights and |errors| through it (*rc != 0: the sample failed)
    BatchSrc per_source(uint64_t seed, int B, const BatchSrc &src, cudaStream_t st, int *rc);
    // ReplayTree.batch_update of that batch, once the update has written the |errors| to the scratch
    int per_write_back(int B, cudaStream_t st) { return per_set(B, per.dev.idx, nullptr, per.dev.abs_err, 1, st); }
};

// The checks and calls of the prioritised-replay entry points (uavrl_per_*, uavrl_sac_per_*) on a handle's store; rs is null
// when the handle is.  Each refuses a store without trees
int per_entry_set(ReplayStore *rs, int device, int32_t n, const int32_t *slots, const double *prio, const float *abs_err, int32_t clip,
                  cudaStream_t st);
int per_entry_sample(ReplayStore *rs, int device, uint64_t seed, int32_t B, const double *u_tape, int32_t *slots, float *w, cudaStream_t st);
int per_entry_get(ReplayStore *rs, int device, double *leaves, double *total, double *beta);

}  // namespace uavrl
