// replay.cu -- the replay store shared by the Q-network and SAC learners (replay.cuh): allocation, batch sources, the lockstep
// iteration and the host read-back.
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
    if ((rc = dev_alloc(&frames, rows * in)) || (rc = pair_actions ? dev_alloc(&act2, 2 * (size_t)slots) : dev_alloc(&act, (size_t)slots)) ||
        (rc = dev_alloc(&rew, (size_t)slots)) || (rc = dev_alloc(&done, (size_t)slots)))
        return rc;
    return 0;
}

void ReplayStore::release()
{
    cudaFree(frames); cudaFree(act); cudaFree(act2); cudaFree(rew); cudaFree(done);
    frames = nullptr; act = nullptr; act2 = nullptr; rew = nullptr; done = nullptr;
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

void ReplayStore::commit()
{
    head = (head + 1) % ring_frames;
    count = count_after_commit();
}

int64_t ReplayStore::count_after_commit() const
{
    const int64_t max_count = (ring_frames - 1) * N;
    return (count + N > max_count) ? max_count : count + N;
}

void ReplayStore::restart()
{
    count = 0;
    frame0_valid = false;
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
    struct Free { void **p[7]; ~Free() { for (auto q : p) if (*q) cudaFree(*q); } } guard{ { (void **)&d_idx, (void **)&d_s, (void **)&d_s2,
                                                                                             (void **)&d_a, (void **)&d_a2, (void **)&d_r, (void **)&d_d } };
    UAVRL_CUDA(cudaMalloc((void **)&d_idx, (size_t)n * 8));
    UAVRL_CUDA(cudaMemcpy(d_idx, idx, (size_t)n * 8, cudaMemcpyHostToDevice));
    if (s) UAVRL_CUDA(cudaMalloc((void **)&d_s, (size_t)n * in * 4));
    if (s2) UAVRL_CUDA(cudaMalloc((void **)&d_s2, (size_t)n * in * 4));
    if (a) UAVRL_CUDA(cudaMalloc((void **)&d_a, (size_t)n * 4));
    if (a2) UAVRL_CUDA(cudaMalloc((void **)&d_a2, (size_t)n * 2 * 4));
    if (r) UAVRL_CUDA(cudaMalloc((void **)&d_r, (size_t)n * 4));
    if (d) UAVRL_CUDA(cudaMalloc((void **)&d_d, (size_t)n));
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
