// replay.cu -- the replay store shared by the Q-network and SAC learners (replay.cuh): allocation, batch sources, the paired
// push, the lockstep iteration and the host read-back.  The prioritised-replay trees follow every change of the store here;
// their operations are in per.cu.
#include "replay.cuh"

namespace uavrl {

// ReplayStore::gather: logical indices -> packed rows (one warp per transition)
__global__ void replay_gather_kernel(int n, int in, BatchSrc src, const int64_t *__restrict__ idx, float *__restrict__ s,
                                     float *__restrict__ s2, int32_t *__restrict__ a, float *__restrict__ a2, float *__restrict__ r,
                                     uint8_t *__restrict__ d)
{
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n) return;
    const ReplayRef t = replay_ref(src, (uint64_t)idx[i]);
    for (int k = lane; k < in; k += 32) {
        if (s) s[(size_t)i * in + k] = src.frames[(size_t)t.row * in + k];
        if (s2) s2[(size_t)i * in + k] = src.frames[(size_t)t.row2 * in + k];
    }
    if (lane == 0) {
        if (a) a[i] = src.act[t.slot];
        if (a2) { a2[2 * i] = src.act2[2 * t.slot]; a2[2 * i + 1] = src.act2[2 * t.slot + 1]; }
        if (r) r[i] = src.rew[t.slot];
        if (d) d[i] = src.done_u8[t.slot];
    }
}

// ReplayStore::push (paired rows)
__global__ void push_kernel(int n, int in, int64_t head, int64_t cap, const float *__restrict__ obs,
                            const int32_t *__restrict__ act, const float *__restrict__ rew,
                            const float *__restrict__ next_obs, const uint8_t *__restrict__ done,
                            float *__restrict__ frames, int32_t *__restrict__ r_act, float *__restrict__ r_rew,
                            uint8_t *__restrict__ r_done)
{
    const int64_t total = (int64_t)n * in;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i / in, k = i - t * in;
        const int64_t slot = (head + t) % cap;
        frames[(2 * slot) * in + k] = obs[i];
        frames[(2 * slot + 1) * in + k] = next_obs[i];
        if (k == 0) { r_act[slot] = act[t]; r_rew[slot] = rew[t]; r_done[slot] = done[t]; }
    }
}

int ReplayStore::alloc(int64_t capacity, int32_t n_envs, int32_t n_trainers, int32_t in, bool pair_actions)
{
    N = n_envs; G = n_trainers; in_dim = in;
    size_t rows;
    if (N > 0) {
        const int64_t Ng = N / G, cap_g = capacity / G;
        int64_t cap_frames = (cap_g + Ng - 1) / Ng;
        if (cap_frames < 2) cap_frames = 2;
        mode = kReplayLockstep;
        ring_frames = cap_frames + 1;
        slots = ring_frames * N;
        rows = (size_t)slots;
    } else {
        mode = kReplayPaired;
        slots = capacity;
        rows = 2 * (size_t)slots;
    }
    int rc;
    if ((rc = mem.alloc(frames, rows * in)) || (rc = pair_actions ? mem.alloc(act2, 2 * (size_t)slots) : mem.alloc(act, (size_t)slots)) ||
        (rc = mem.alloc(rew, (size_t)slots)) || (rc = mem.alloc(done, (size_t)slots)))
        return rc;
    return 0;
}

BatchSrc ReplayStore::source(uint64_t seed, int64_t epoch, const int32_t *idx_tape) const
{
    BatchSrc s;
    memset(&s, 0, sizeof(s));
    s.mode = mode; s.frames = frames; s.act = act; s.act2 = act2; s.rew = rew; s.done_u8 = done;
    s.idx_tape = idx_tape; s.count = count;
    s.key = seed ^ kSampleSalt; s.epoch = (uint64_t)epoch;
    if (mode == kReplayLockstep) {
        // every trainer samples its own block of N / G envs (trainer_src), count = its transitions
        s.cap = ring_frames; s.n_envs = N / G; s.row_stride = N;
        s.count = count / G;
        s.oldest = ((head - count / N) % ring_frames + ring_frames) % ring_frames;
    } else {
        s.cap = slots;
        s.oldest = ((head - count) % slots + slots) % slots;
    }
    return s;
}

int ReplayStore::push(int32_t n, const float *obs, const int32_t *a, const float *r, const float *next_obs, const uint8_t *d,
                      cudaStream_t st)
{
    const int64_t total = (int64_t)n * in_dim;
    const int threads = 256;
    int blocks = (int)((total + threads - 1) / threads);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    push_kernel<<<blocks, threads, 0, st>>>(n, in_dim, head, slots, obs, a, r, next_obs, d, frames, act, rew, done);
    UAVRL_LAUNCHED();
    if (per_enabled()) {                                          // ReplayTree.push with error 0; uavrl_per_set_errors refines it
        int rc = per_fill_range(head, n, per.new_priority(), st);
        if (rc) return rc;
    }
    head = (head + n) % slots;
    count = (count + n > slots) ? slots : count + n;
    return 0;
}

ReplayStore::Iteration ReplayStore::begin() const
{
    const int64_t f = head, fn = (head + 1) % ring_frames;
    Iteration it;
    it.obs_t = frames + f * N * in_dim;
    it.obs_next = frames + fn * N * in_dim;
    it.act = act ? act + f * N : nullptr;
    it.act2 = act2 ? act2 + 2 * f * N : nullptr;
    it.rew = rew + f * N; it.done = done + f * N;
    return it;
}

int ReplayStore::commit(cudaStream_t st)
{
    if (per_enabled()) {
        // the frame just completed becomes sampleable with the priority of an error-less push; the frame that now
        // receives the next observations (the ring's oldest) stops being a transition.  Trainer-local slots: every trainer's
        // tree gets the same Ng + Ng slots of its own env block
        const int64_t Ng = N / G;
        if (int rc = per_fill_range(head * Ng, 2 * Ng, per.new_priority(), st, Ng, 0.0)) return rc;
    }
    head = (head + 1) % ring_frames;
    count = count_after_commit();
    return 0;
}

int64_t ReplayStore::count_after_commit() const
{
    const int64_t max_count = (ring_frames - 1) * N;
    return (count + N > max_count) ? max_count : count + N;
}

int ReplayStore::restart()
{
    count = 0;
    frame0_valid = false;
    return per_clear();
}

int ReplayStore::gather(int32_t n, const int64_t *idx, float *s, int32_t *a, float *a2, float *r, float *s2, uint8_t *d) const
{
    for (int i = 0; i < n; ++i)
        if (idx[i] < 0 || idx[i] >= count) return fail(UAVRL_ERR_INVALID, "logical index out of range");
    UAVRL_CUDA(cudaDeviceSynchronize());
    BatchSrc src = source(0, 0, nullptr);
    if (mode == kReplayLockstep) src.n_envs = src.row_stride;      // whole-ring logical indices, whatever the trainer count
    const size_t in = (size_t)in_dim;
    // one gather kernel into a packed staging block, then one device->host copy per output array
    int64_t *d_idx = nullptr; float *d_s = nullptr, *d_s2 = nullptr, *d_a2 = nullptr, *d_r = nullptr; int32_t *d_a = nullptr; uint8_t *d_d = nullptr;
    DevMem m;
    int rc;
    if ((rc = m.alloc(d_idx, (size_t)n, false))) return rc;
    UAVRL_CUDA(cudaMemcpy(d_idx, idx, (size_t)n * 8, cudaMemcpyHostToDevice));
    if ((s && (rc = m.alloc(d_s, (size_t)n * in, false))) || (s2 && (rc = m.alloc(d_s2, (size_t)n * in, false))) ||
        (a && (rc = m.alloc(d_a, (size_t)n, false))) || (a2 && (rc = m.alloc(d_a2, (size_t)n * 2, false))) ||
        (r && (rc = m.alloc(d_r, (size_t)n, false))) || (d && (rc = m.alloc(d_d, (size_t)n, false))))
        return rc;
    replay_gather_kernel<<<(n + 7) / 8, 256>>>(n, (int)in, src, d_idx, d_s, d_s2, d_a, d_a2, d_r, d_d);
    UAVRL_CUDA(cudaGetLastError());
    if (s) UAVRL_CUDA(cudaMemcpy(s, d_s, (size_t)n * in * 4, cudaMemcpyDeviceToHost));
    if (s2) UAVRL_CUDA(cudaMemcpy(s2, d_s2, (size_t)n * in * 4, cudaMemcpyDeviceToHost));
    if (a) UAVRL_CUDA(cudaMemcpy(a, d_a, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (a2) UAVRL_CUDA(cudaMemcpy(a2, d_a2, (size_t)n * 2 * 4, cudaMemcpyDeviceToHost));
    if (r) UAVRL_CUDA(cudaMemcpy(r, d_r, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (d) UAVRL_CUDA(cudaMemcpy(d, d_d, (size_t)n, cudaMemcpyDeviceToHost));
    return 0;
}

}  // namespace uavrl
