// wgmma.cuh -- Hopper (sm_90a) warpgroup tensor-core helpers, inline PTX: shared-memory matrix descriptors (K-major, no
// swizzle), wgmma.mma_async kind tf32 with fp32 accumulation in registers, and the 3xTF32 split products the kernels use.
//
// Operand layout used throughout (canonical K-major "interleave" layout, no swizzle):
//   core matrix = 8 rows x 16 bytes (4 fp32/tf32 values), stored as 128 contiguous bytes (row stride 16 B);
//   core matrices adjacent in K are LBO bytes apart, adjacent in M/N (next 8 rows) SBO bytes apart.
//   element (r, c) of a [rows][K] operand lives at   (r/8)*SBO + (c/4)*LBO + (r%8)*16 + (c%4)*4.
//   One tf32 wgmma consumes K = 8 (two 16-byte chunks); the next K step starts 2*LBO further.
// wgmma reads tf32 operands from shared memory K-major only, so every product contracts over the operands' fast index.
//
// Accumulators: a warpgroup (128 threads) owns an m64 x N fp32 tile in registers; mma_3xtf32 stages it through a
// row-major shared-memory tile; the elementwise epilogues read it in 4-column groups spread over every thread (EpiSlice), the
// head epilogues one sample row (32 consecutive columns) per thread.
#pragma once
#include <stdint.h>

namespace uavrl {

constexpr uint32_t kMmaLBO = 128;                  // K-adjacent core matrices are contiguous

__host__ __device__ constexpr uint32_t mma_sbo(int k_pad) { return (uint32_t)(k_pad / 4) * 128u; }
__host__ __device__ constexpr uint32_t mma_tile_bytes(int rows, int k_pad) { return (uint32_t)(rows / 8) * mma_sbo(k_pad); }

// byte offset of element (r, c) inside an operand tile
__device__ __forceinline__ uint32_t mma_off(int r, int c, uint32_t sbo, uint32_t lbo = kMmaLBO)
{
    return (uint32_t)(r >> 3) * sbo + (uint32_t)(c >> 2) * lbo + (uint32_t)(r & 7) * 16u + (uint32_t)(c & 3) * 4u;
}

// 64-bit wgmma shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset 0,
// layout type 0 (no swizzle) [62,64)
__device__ __forceinline__ uint64_t mma_desc(const void *smem_ptr, uint32_t sbo, uint32_t lbo = kMmaLBO)
{
    const uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
    uint64_t d = 0;
    d |= (uint64_t)((addr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo >> 4) & 0x3FFFu) << 32;
    return d;
}

// 3xTF32 split: hi = x rounded to TF32 (10-bit mantissa), lo = x - hi (exact).  hi*hi + hi*lo + lo*hi
// reproduces the fp32 product to ~2^-21.
// Round-to-nearest, ties away (cvt.rna.tf32.f32) on the bit pattern: add half an ulp of the 10-bit mantissa to the magnitude
// and clear the 13 dropped bits -- two integer instructions.  ptxas expands the cvt into the same two plus an |x| < inf
// test and a select per element (inf/NaN kept verbatim); for every finite x that does not round up to inf the result is
// bit-identical, inf stays inf, and the epilogues run this 32 times per thread per layer.
__device__ __forceinline__ void tf32_split(float x, float &hi, float &lo)
{
    hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
    lo = x - hi;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void fence_operands(float *d)
{
#pragma unroll
    for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, both operands K-major in shared memory; the whole warpgroup issues.
// scale_d == 0 overwrites D.  Thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns
// 8*i + 2*(t%4) (+1): d[4i] (r, c), d[4i+1] (r, c+1), d[4i+2] (r+8, c), d[4i+3] (r+8, c+1).
template <int N> __device__ __forceinline__ void wgmma_tf32(float *d, uint64_t a, uint64_t b, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_tf32<16>(float *d, uint64_t a, uint64_t b, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float *d, uint64_t a, uint64_t b, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float *d, uint64_t a, uint64_t b, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(scale_d));
}

// The three TF32 products hi*hi + hi*lo + lo*hi of one K extent (K = 8 * ksteps) into the warpgroup's registers.
// accumulate == 0: the first product overwrites d.  The next K step is +2*LBO bytes = +16 in the descriptor's address field.
// With a runtime ksteps ptxas closes the wgmma group every few instructions and re-opens it (C7519: warpgroup.arrive injected),
// so the layer products of the shipped networks use wgmma_3xtf32_k below; this one serves compile-time K (tc_dw_kernel)
// and every other network shape.
template <int N>
__device__ __forceinline__ void wgmma_3xtf32(float *d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, int ksteps,
                                             uint32_t accumulate)
{
    const uint64_t kStep = (uint64_t)((2 * kMmaLBO) >> 4);
    fence_operands<N>(d);
    wgmma_fence();
    for (int k = 0; k < ksteps; ++k) wgmma_tf32<N>(d, a_hi + k * kStep, b_hi + k * kStep, (k > 0 || accumulate) ? 1u : 0u);
    for (int k = 0; k < ksteps; ++k) wgmma_tf32<N>(d, a_hi + k * kStep, b_lo + k * kStep, 1u);
    for (int k = 0; k < ksteps; ++k) wgmma_tf32<N>(d, a_lo + k * kStep, b_hi + k * kStep, 1u);
    wgmma_commit();
    wgmma_wait0();
    fence_operands<N>(d);
}

// The same products for a compile-time K extent (K = 8 * KS): all 3 * KS wgmma back to back behind one fence, one commit,
// one wait -- one unbroken chain.
template <int N, int KS>
__device__ __forceinline__ void wgmma_3xtf32_k(float *d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo)
{
    const uint64_t kStep = (uint64_t)((2 * kMmaLBO) >> 4);
    fence_operands<N>(d);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k) wgmma_tf32<N>(d, a_hi + k * kStep, b_hi + k * kStep, k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < KS; ++k) wgmma_tf32<N>(d, a_hi + k * kStep, b_lo + k * kStep, 1u);
#pragma unroll
    for (int k = 0; k < KS; ++k) wgmma_tf32<N>(d, a_lo + k * kStep, b_hi + k * kStep, 1u);
    wgmma_commit();
    wgmma_wait0();
    fence_operands<N>(d);
}

// Which layer product a call site issues: the forward chain (A = activations, B = W) or the dX chain (A = dZ, B = W^T).
enum MmaKind { kMmaFwd = 0, kMmaDx = 1 };

// The (chunk width, k-steps) pairs of the shipped networks (input 100, hidden 64 / 128, head 27 / 28 padded to 32), which the
// kernels issue as compile-time chains: forward 64-column chunks over the input (13) or a 64 / 128-wide hidden layer (8 / 16)
// and the 32-column head over a 64-wide hidden layer (8); dX 64-column chunks over the head's 32 or a hidden layer's 64
// gradients (4 / 8).  Only these pairs, so that each call site carries a few chains and not every combination.
__host__ __device__ constexpr bool mma_fixed(int kind, int n, int ksteps)
{
    return kind == kMmaFwd ? (n == 64 && (ksteps == 13 || ksteps == 8 || ksteps == 16)) || (n == 32 && ksteps == 8)
                           : n == 64 && (ksteps == 4 || ksteps == 8);
}
// every chunk of an N-wide product (64-column chunks, then 32, then 16) is one of the pairs above
__host__ __device__ constexpr bool mma_fixed_product(int kind, int n, int ksteps)
{
    return (n < 64 || mma_fixed(kind, 64, ksteps)) && (n % 64 < 32 || mma_fixed(kind, 32, ksteps)) && n % 32 == 0;
}

template <int N, int KIND>
__device__ __forceinline__ void wgmma_3xtf32_fixed(float *d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, int ksteps)
{
    if constexpr (mma_fixed(KIND, N, 4)) if (ksteps == 4) wgmma_3xtf32_k<N, 4>(d, a_hi, a_lo, b_hi, b_lo);
    if constexpr (mma_fixed(KIND, N, 8)) if (ksteps == 8) wgmma_3xtf32_k<N, 8>(d, a_hi, a_lo, b_hi, b_lo);
    if constexpr (mma_fixed(KIND, N, 13)) if (ksteps == 13) wgmma_3xtf32_k<N, 13>(d, a_hi, a_lo, b_hi, b_lo);
    if constexpr (mma_fixed(KIND, N, 16)) if (ksteps == 16) wgmma_3xtf32_k<N, 16>(d, a_hi, a_lo, b_hi, b_lo);
}

// the warpgroup's fragment -> acc[row][col0 + c] (row-major, ld floats per row); rows >= R are not stored
template <int N>
__device__ __forceinline__ void store_frag(const float *d, float *acc, int ld, int row0, int col0, int R)
{
    const int t = threadIdx.x & 127, r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = col0 + 2 * (t & 3);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
        if (r < R) *reinterpret_cast<float2 *>(acc + (size_t)r * ld + c + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
        if (r + 8 < R) *reinterpret_cast<float2 *>(acc + (size_t)(r + 8) * ld + c + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
}

// FIXED: the product is one of the pairs above (mma_fixed_product), issued as one unbroken chain.  Otherwise the runtime-K
// chain; a kernel that has it anywhere gets every chain broken up by ptxas, so the kernels come in both variants
// and the host picks the FIXED one whenever the network's shape allows.
template <int N, int KIND, bool FIXED>
__device__ __forceinline__ void mma_chunk(float *acc, int ld, int row0, int n0, uint64_t a_hi, uint64_t a_lo, const unsigned char *b_hi,
                                          const unsigned char *b_lo, uint32_t sbo, int ksteps, int R)
{
    float d[N / 2];
    // The runtime-K chain's first product overwrites d only through a runtime scale-d predicate, so to ptxas d is read
    // before it is written.  Left undefined, its registers may get a definition placed inside the wgmma pipeline stage,
    // depending on the surrounding code, and ptxas then serialises every wgmma of the kernel (C7515).  Zeroing d ahead of
    // the fence rules that out; the products are unchanged.
    if (!FIXED) {
#pragma unroll
        for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    }
    const uint32_t boff = (uint32_t)(n0 >> 3) * sbo;
    const uint64_t bh = mma_desc(b_hi + boff, sbo), bl = mma_desc(b_lo + boff, sbo);
    if (FIXED) wgmma_3xtf32_fixed<N, KIND>(d, a_hi, a_lo, bh, bl, ksteps);
    else wgmma_3xtf32<N>(d, a_hi, a_lo, bh, bl, ksteps, 0u);
    store_frag<N>(d, acc, ld, row0, n0, R);
}

// acc[r][c] = sum_k A[r][k] * B[c][k] in 3xTF32 for r < R, c < N (N a multiple of 16), K = 8 * ksteps; A and B share the
// K extent and so the SBO.  Called by every thread of the CTA (256 = two warpgroups, warpgroup g computes rows [64g, 64g + 64),
// and only where they hold real rows); ends with a CTA barrier behind which acc is complete.  The operands' generic-proxy
// writes must have been fenced (fence_proxy_async) and published by a barrier before the call.
template <int KIND, bool FIXED>
__device__ __forceinline__ void mma_3xtf32(float *acc, int ld, const unsigned char *a_hi, const unsigned char *a_lo,
                                           const unsigned char *b_hi, const unsigned char *b_lo, uint32_t sbo, int N, int ksteps, int R)
{
    const int row0 = (threadIdx.x >> 7) * 64;
    if (row0 < R) {
        const uint64_t ah = mma_desc(a_hi + (row0 >> 3) * sbo, sbo), al = mma_desc(a_lo + (row0 >> 3) * sbo, sbo);
        int n0 = 0;
        for (; n0 + 64 <= N; n0 += 64) mma_chunk<64, KIND, FIXED>(acc, ld, row0, n0, ah, al, b_hi, b_lo, sbo, ksteps, R);
        if (n0 + 32 <= N) { mma_chunk<32, KIND, FIXED>(acc, ld, row0, n0, ah, al, b_hi, b_lo, sbo, ksteps, R); n0 += 32; }
        if (!FIXED && n0 < N) mma_chunk<16, KIND, FIXED>(acc, ld, row0, n0, ah, al, b_hi, b_lo, sbo, ksteps, R);
    }
    __syncthreads();
}

// row `row` of the staged accumulator, columns [c0, c0 + 32)
__device__ __forceinline__ void acc_ld32(const float *acc, int ld, int row, int c0, float (&v)[32])
{
    const float4 *src = reinterpret_cast<const float4 *>(acc + (size_t)row * ld + c0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 t = src[j];
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
}

// One thread's share of an elementwise epilogue over the staged R x N accumulator (R = 32 / 64 / 128 rows, nt threads): row
// t % R, 4-column groups c0, c0 + step, ... (c0 = 4 * (t / R), step = 4 * nt / R).  Every warp of the CTA, on all four
// scheduler sub-partitions, takes part whatever R is.  Eight consecutive lanes read eight rows of one group (ld = 4 mod 32
// words: no bank conflict) and write one whole core matrix of the next A operand (128 contiguous bytes).
struct EpiSlice {
    int row, c0, step;
    __device__ __forceinline__ EpiSlice(int R, int nt)
    {
        const int lgR = 31 - __clz(R);
        row = threadIdx.x & (R - 1); c0 = 4 * (threadIdx.x >> lgR); step = 4 * (nt >> lgR);
    }
    __device__ __forceinline__ float4 ld(const float *acc, int ld, int c) const
    {
        return *reinterpret_cast<const float4 *>(acc + (size_t)row * ld + c);
    }
};

}  // namespace uavrl
