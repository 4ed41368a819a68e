// tc_chain.cuh -- the Q-network forward chain on the tensor cores, shared by the act / TD / federation-loss kernels
// (tc_forward.cu) and the training kernel with its fused TD pre-pass (tc_train.cu): the layer-0 gather, the hidden-layer
// epilogue, the layer loop, the Q head and the staging of the forward weight image.
#pragma once
#include "tc_forward.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace uavrl {

// UAVRL_TC_TRACE=1: CTA (cta, 0) / thread 0 writes clock64() to slot `slot` at a stage boundary (stage_trace_print reads them)
__device__ __forceinline__ void stage_trace(long long *t, int slot, int cta = 0)
{
    if (t && blockIdx.x == cta && blockIdx.y == 0 && threadIdx.x == 0) t[slot] = clock64();
}

// ---- A operand of layer 0: R gathered rows -> TF32 hi/lo, canonical K-major layout.  Item i = (chunk j = i / R, row r = i % R;
// R is a power of two): consecutive lanes take consecutive rows of the same 16-byte chunk, so a quarter-warp's 16-byte stores
// cover one whole core-matrix column = 128 contiguous bytes (lanes walking along a row would all hit the same 4 banks) and the
// index needs no division.  A thread handles items i0 + u * kTcThreads, u < 4, and issues all four loads before it converts
// any, so the gather costs one L2 round trip.  row_of(r) is row r's input vector (nullptr: a zero row): obs + row * in_dim in
// the act pass, a row-pointer table elsewhere.
template <class RowOf>
__device__ __forceinline__ void a0_load(const RowOf &row_of, int i0, int R, int in_dim, int K0, float4 (&v)[4])
{
    const int total = R * (K0 / 4), lgR = 31 - __clz(R);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kTcThreads;
        const int r = i & (R - 1), j = i >> lgR;
        const float *rp = (i < total) ? row_of(r) : nullptr;
        v[u] = (rp && 4 * j < in_dim) ? __ldg(reinterpret_cast<const float4 *>(rp) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}
// The load half for a tile whose next-state rows are partly being written by the predecessor: want_fresh = false loads every
// row NOT flagged in fresh[] (everything else zero) and may run before the dependent-launch wait; want_fresh = true then loads
// only the flagged rows, from L2, into the same registers.
__device__ __forceinline__ void a0_load_sel(const float *const *rows, const uint8_t *fresh, bool want_fresh, int R, int in_dim, int K0, float4 (&v)[4])
{
    const int total = R * (K0 / 4), lgR = 31 - __clz(R);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int i = threadIdx.x + u * kTcThreads;
        const int r = i & (R - 1), j = i >> lgR;
        const float *rp = (i < total) ? rows[r] : nullptr;
        const bool take = rp && 4 * j < in_dim && ((fresh[r] != 0) == want_fresh);
        if (!want_fresh) v[u] = take ? __ldg(reinterpret_cast<const float4 *>(rp) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
        else if (take) v[u] = __ldcg(reinterpret_cast<const float4 *>(rp) + j);
    }
}
__device__ __forceinline__ void a0_store(const float4 (&v)[4], int i0, int R, int K0, unsigned char *Ahi, unsigned char *Alo)
{
    const int total = R * (K0 / 4), lgR = 31 - __clz(R);
    const uint32_t sbo = mma_sbo(K0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kTcThreads;
        if (i < total) {
            const int r = i & (R - 1), j = i >> lgR;
            float4 h, l;
            tf32_split(v[u].x, h.x, l.x); tf32_split(v[u].y, h.y, l.y); tf32_split(v[u].z, h.z, l.z); tf32_split(v[u].w, h.w, l.w);
            const uint32_t off = mma_off(r, 4 * j, sbo);
            *reinterpret_cast<float4 *>(Ahi + off) = h;
            *reinterpret_cast<float4 *>(Alo + off) = l;
        }
    }
}
// the whole gather: load and store halves over every item of the tile
template <class RowOf>
__device__ __forceinline__ void a0_gather(const RowOf &row_of, int R, int in_dim, int K0, unsigned char *Ahi, unsigned char *Alo)
{
    for (int i0 = threadIdx.x; i0 < R * (K0 / 4); i0 += 4 * kTcThreads) {
        float4 v[4];
        a0_load(row_of, i0, R, in_dim, K0, v);
        a0_store(v, i0, R, K0, Ahi, Alo);
    }
}

// ---- hidden-layer epilogue over this thread's EpiSlice of the staged N-column accumulator: bias + ReLU, TF32 re-split into the
// next layer's A operand (K = N).  KEEP (training chain): the activations also go to act_row (when `mine`: a real sample) for
// the weight gradients, and the result is the ReLU mask for the dX chain, bit 4i + j = (H[e.row][e.c0 + i * e.step + j] > 0).
template <bool KEEP>
__device__ __forceinline__ uint32_t hidden_epilogue(const EpiSlice &e, const float *acc, int acc_ld, const float *bias, int N,
                                                    unsigned char *Ahi, unsigned char *Alo, float *act_row, bool mine)
{
    const uint32_t sbon = mma_sbo(N);
    uint32_t mk = 0u;
    for (int c = e.c0, sh = 0; c < N; c += e.step, sh += 4) {
        const float4 v = e.ld(acc, acc_ld, c);
        float4 x, h, lo4;
        x.x = fmaxf(v.x + bias[c + 0], 0.f); x.y = fmaxf(v.y + bias[c + 1], 0.f);
        x.z = fmaxf(v.z + bias[c + 2], 0.f); x.w = fmaxf(v.w + bias[c + 3], 0.f);
        tf32_split(x.x, h.x, lo4.x); tf32_split(x.y, h.y, lo4.y); tf32_split(x.z, h.z, lo4.z); tf32_split(x.w, h.w, lo4.w);
        const uint32_t off = mma_off(e.row, c, sbon);
        *reinterpret_cast<float4 *>(Ahi + off) = h;
        *reinterpret_cast<float4 *>(Alo + off) = lo4;
        if (KEEP) {
            if (mine) *reinterpret_cast<float4 *>(act_row + c) = x;
            mk |= ((x.x > 0.f ? 1u : 0u) | (x.y > 0.f ? 2u : 0u) | (x.z > 0.f ? 4u : 0u) | (x.w > 0.f ? 8u : 0u)) << sh;
        }
    }
    return mine ? mk : 0u;
}

// ---- Q head: a 32-wide padded row q of the head accumulator plus the bias; DUELING: Q = V + A - mean(A) with V in column nA
// (BaseCNN.py:138)
template <bool DUELING>
__device__ __forceinline__ void q_combine(const float *bias, int nA, float (&q)[32])
{
#pragma unroll
    for (int j = 0; j < 32; ++j) q[j] += bias[j];
    if (DUELING) {
        float s = 0.f, V = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) { if (j < nA) s += q[j]; if (j == nA) V = q[j]; }
        const float mean = s / (float)nA;
#pragma unroll
        for (int j = 0; j < 32; ++j) q[j] = V + q[j] - mean;
    }
}
// ... of row `row` of the staged head accumulator
template <bool DUELING>
__device__ __forceinline__ void q_row(const float *acc, int acc_ld, int row, const float *bias, int nA, float (&q)[32])
{
    acc_ld32(acc, acc_ld, row, 0, q);
    q_combine<DUELING>(bias, nA, q);
}
// the first maximum over the nA actions, its value in bv
__device__ __forceinline__ int q_argmax(const float (&q)[32], int nA, float &bv)
{
    int best = 0;
    bv = q[0];
#pragma unroll
    for (int j = 1; j < 32; ++j) if (j < nA && q[j] > bv) { bv = q[j]; best = j; }
    return best;
}
// q[a] by a select over the registers (no local-memory indexing)
__device__ __forceinline__ float q_at(const float (&q)[32], int a)
{
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) if (j == a) v = q[j];
    return v;
}

// ---- staging: the forward image travels in two pieces, layer 0's hi|lo block on wbar (all the first product needs) and the
// other layers with the biases on wbar2, which the callers first wait for behind layer 0's product.  Where the image can only
// be requested after the dependent-launch wait, half of its latency is then covered by the first layer.
__device__ __forceinline__ uint32_t fwd_image_split(const TcNet &tc) { return tc.n_layers > 1 ? (uint32_t)tc.L[1].hi_off : (uint32_t)tc.img_bytes; }
__device__ __forceinline__ void stage_forward_image(const TcNet &tc, unsigned char *W, const unsigned char *img, uint64_t *wbar, uint64_t *wbar2)
{
    const uint32_t split = fwd_image_split(tc);
    fence_proxy_async();
    bulk_g2s_chunked(W, img, split, wbar);
    if (split < (uint32_t)tc.img_bytes) bulk_g2s_chunked(W + split, img + split, (uint32_t)tc.img_bytes - split, wbar2);
}

// ---- one forward pass over the network for a tile of R rows whose layer-0 operand is in place.  Per layer: the product
// (mma_3xtf32, ends with a CTA barrier), mid(l) (the caller's waits and trace marks), then either the hidden-layer epilogue,
// fence and barrier, done(l, ReLU mask) -- or, for the last layer, head(l, bias), which writes the caller's outputs and ends
// with whatever barrier the caller needs.  KEEP: the epilogues also store the activations (hidden_epilogue), layer l + 1's
// input at act_row + L[l + 1].act_off.
template <bool FIXED, bool KEEP, class Mid, class Head, class Done>
__device__ __forceinline__ void forward_layers(const TcNet &tc, int R, const EpiSlice &e, unsigned char *Ahi, unsigned char *Alo,
                                               const unsigned char *W, float *acc, float *act_row, bool mine, Mid &&mid, Head &&head,
                                               Done &&done)
{
    const float *bias_all = reinterpret_cast<const float *>(W + tc.bias_base);
    for (int l = 0; l < tc.n_layers; ++l) {
        const TcLayer T = tc.L[l];
        mma_3xtf32<kMmaFwd, FIXED>(acc, tc.acc_ld, Ahi, Alo, W + T.hi_off, W + T.lo_off, mma_sbo(T.K_pad), T.N_pad, T.K_pad / 8, R);
        mid(l);
        const float *bias = bias_all + T.bias_off;
        if (l + 1 < tc.n_layers) {
            const uint32_t mk = hidden_epilogue<KEEP>(e, acc, tc.acc_ld, bias, T.N_pad, Ahi, Alo, KEEP ? act_row + tc.L[l + 1].act_off : nullptr, mine);
            fence_proxy_async();
            __syncthreads();
            done(l, mk);
        } else {
            head(l, bias);
        }
    }
}

}  // namespace uavrl
