// common.cuh -- error plumbing, launch accounting and the counter-based RNG shared by the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/uavrl.h"
#include "launch_chain.cuh"

namespace uavrl {

extern thread_local std::string g_last_error;

// streaming multiprocessors of the current device (132 on an H100 SXM): grid sizes of the one-wave kernels and tile-size
// thresholds are derived from it, so a part with fewer SMs keeps the one-wave sizing.  Read once per device.
inline int num_sms()
{
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
extern std::atomic<long long> g_launches;

// shared memory one block may use on sm_90 (dynamic + static): every kernel that keeps a network resident is sized against it
constexpr size_t kMaxBlockSmem = 227 * 1024;

inline int fail(int code, const std::string &msg)
{
    g_last_error = msg;
    return code;
}

#define UAVRL_CUDA(expr)                                                                      \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            char _b[512];                                                                     \
            snprintf(_b, sizeof(_b), "%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,      \
                     cudaGetErrorString(_e));                                                 \
            return ::uavrl::fail(UAVRL_ERR_CUDA, _b);                                         \
        }                                                                                     \
    } while (0)

#define UAVRL_LAUNCHED()                                                                      \
    do {                                                                                      \
        ::uavrl::g_launches.fetch_add(1, std::memory_order_relaxed);                          \
        UAVRL_CUDA(cudaGetLastError());                                                       \
    } while (0)

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------------------
// Inside the lockstep loops every kernel depends on its predecessor, so each kernel boundary would cost a full
// drain + launch + prologue.  Kernels of the loop are launched with programmaticStreamSerialization: a CTA of
// kernel k+1 may start while kernel k is still running, does what does not depend on k (mbarrier init, TMA of weights / loads of state last written >= 2 kernels back) and then blocks in griddepcontrol.wait
// until k has completed and its writes are visible.  Every loop kernel triggers its dependents right after its own
// wait, so kernel k+1 only ever overlaps kernel k (everything <= k-1 is complete when k+1's prologue runs).
// Launched without the attribute, both instructions are no-ops.  Which kernel launches so, and what it may fetch before its
// wait, is decided in launch_chain.cuh.

#if defined(__CUDACC__)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                                 Args... args)
{
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the kernel (process-wide, per device), not to the learner that sets
// it: raise it to what this instance launches with, never lower it.  Setting it to a smaller instance's size would make every
// launch of a larger instance that is still alive fail.
template <class K>
inline int raise_dyn_smem(K *kernel, size_t bytes)
{
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    cudaFuncAttributes fa;
    UAVRL_CUDA(cudaFuncGetAttributes(&fa, kernel));
    if ((size_t)fa.maxDynamicSharedSizeBytes < bytes)
        UAVRL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return 0;
}

extern std::atomic<int> g_fail_alloc;    // uavrl_test_fail_alloc(); -1 = off

// Owner of a group of device buffers that live and die together: every pointer alloc() hands out is freed by release() or the
// destructor.  Host handles hold one DevMem per group; the kernel-argument structs keep plain pointers into them.  A failed
// alloc() leaves p untouched, clears the runtime's error state and returns UAVRL_ERR_CUDA ("out of memory").
class DevMem {
public:
    DevMem() = default;
    DevMem(DevMem &&o) noexcept : ptrs_(std::move(o.ptrs_)) {}
    DevMem &operator=(DevMem &&o) noexcept { if (this != &o) { release(); ptrs_.swap(o.ptrs_); } return *this; }
    ~DevMem() { release(); }
    void release() { for (void *p : ptrs_) cudaFree(p); ptrs_.clear(); }
    // n elements of T, zeroed unless zero = false
    template <class T>
    int alloc(T *&p, size_t n, bool zero = true)
    {
        int k = g_fail_alloc.load(std::memory_order_relaxed);
        while (k >= 0 && !g_fail_alloc.compare_exchange_weak(k, k - 1, std::memory_order_relaxed)) {}
        void *q = nullptr;
        const cudaError_t e = k == 0 ? cudaErrorMemoryAllocation : cudaMalloc(&q, n * sizeof(T));
        if (e != cudaSuccess) {
            cudaGetLastError();                                  // a failed cudaMalloc must not surface at the next launch check
            return fail(UAVRL_ERR_CUDA, "cudaMalloc of " + std::to_string(n * sizeof(T)) + " bytes failed: " + cudaGetErrorString(e));
        }
        ptrs_.push_back(q);
        if (zero) UAVRL_CUDA(cudaMemset(q, 0, n * sizeof(T)));
        p = static_cast<T *>(q);
        return 0;
    }

private:
    std::vector<void *> ptrs_;
};

// Scratch that grows with the batch: when need exceeds cap, wait for st, free the group, then allocate every buffer of bufs
// (pointer, element count) afresh and set cap = need.  On failure the group is empty, every pointer null and cap 0, so the
// next call grows again.
template <class T> struct Buf { T *&p; size_t n; };
template <class T> Buf<T> buf(T *&p, size_t n) { return Buf<T>{ p, n }; }
template <class Cap, class... T>
int grow(DevMem &m, Cap &cap, Cap need, cudaStream_t st, bool zero, Buf<T>... bufs)
{
    if (need <= cap) return 0;
    UAVRL_CUDA(cudaStreamSynchronize(st));
    m.release();
    cap = 0;
    int rc = 0;
    ((rc = rc ? rc : m.alloc(bufs.p, bufs.n, zero)), ...);
    if (rc) {
        m.release();
        ((bufs.p = nullptr), ...);
        return rc;
    }
    cap = need;
    return 0;
}

// Philox4x32-10 (Salmon et al. 2011), counter-based: stream = (key, counter), no state to store.
struct Philox {
    static __host__ __device__ __forceinline__ void round(uint32_t (&c)[4], uint32_t k0, uint32_t k1)
    {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
        const uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
        const uint32_t h0 = (uint32_t)(p0 >> 32), l0 = (uint32_t)p0;
        const uint32_t h1 = (uint32_t)(p1 >> 32), l1 = (uint32_t)p1;
        const uint32_t n0 = h1 ^ c[1] ^ k0, n2 = h0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = l1; c[2] = n2; c[3] = l0;
    }
    static __host__ __device__ __forceinline__ void gen(uint64_t key, uint64_t ctr_lo, uint64_t ctr_hi,
                                                        uint32_t (&out)[4])
    {
        uint32_t c[4] = { (uint32_t)ctr_lo, (uint32_t)(ctr_lo >> 32), (uint32_t)ctr_hi, (uint32_t)(ctr_hi >> 32) };
        uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            round(c, k0, k1);
            k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
        }
        out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
    }
    // uniform in [0,1) with 24 random bits (what a float can hold exactly)
    static __host__ __device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }
};

}  // namespace uavrl
