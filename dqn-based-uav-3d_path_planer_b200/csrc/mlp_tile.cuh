// mlp_tile.cuh -- fp32 CUDA-core building blocks of the SMEM-resident MLP kernels (learner.cu, sac.cu):
// a CTA owns a tile of 32 samples; a whole network is staged transposed in shared memory (Wt[k][o], ld = out|1)
// by one TMA bulk copy of its pre-packed image; lanes walk output units, each warp carries 4 samples.
#pragma once
#include <vector>

#include "net.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace uavrl {

__device__ __forceinline__ int ldw_of(int out) { return (out & 1) ? out : out + 1; }

// flat parameter index -> position in the smem weight image (Wt[k][o] transposed, ld = out|1; biases after)
inline void build_image_map(const NetDev &net, std::vector<int32_t> &map)
{
    map.assign((size_t)net.P, 0);
    for (int l = 0; l < net.n_layers; ++l) {
        const LayerDev &L = net.L[l];
        const int ldw = (L.out & 1) ? L.out : L.out + 1, in = L.in;
        for (int o = 0; o < L.out; ++o) {
            const bool extra = o >= L.out_main;            // rows of the second head block (dueling V / actor sigma)
            const size_t wbase = extra ? (size_t)L.w2_off + (size_t)(o - L.out_main) * in : (size_t)L.w_off + (size_t)o * in;
            for (int k = 0; k < in; ++k) map[wbase + k] = L.smem_w + k * ldw + o;
            map[extra ? (size_t)L.b2_off + (o - L.out_main) : (size_t)L.b_off + o] = L.smem_b + o;
        }
    }
}

// blockIdx.y: network y of a stack of networks ([y][P] parameters, images img_stride floats apart)
static __global__ void pack_image_kernel(int P, const float *__restrict__ flat, const int32_t *__restrict__ map, float *__restrict__ img,
                                         int img_stride)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    flat += (size_t)blockIdx.y * P; img += (size_t)blockIdx.y * img_stride;
    if (i < P) img[map[i]] = flat[i];
}

static __global__ void pack_tc_kernel(int P, const float *__restrict__ flat, const int32_t *__restrict__ hi_map,
                               const int32_t *__restrict__ lo_map, const int32_t *__restrict__ hi2_map,
                               const int32_t *__restrict__ lo2_map, float *__restrict__ img, int img_stride)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    flat += (size_t)blockIdx.y * P; img += (size_t)blockIdx.y * img_stride;
    const float p = flat[i];
    if (lo_map[i] >= 0) {
        float hi, lo; tf32_split(p, hi, lo);
        img[hi_map[i]] = hi; img[lo_map[i]] = lo;
        if (hi2_map[i] >= 0) { img[hi2_map[i]] = hi; img[lo2_map[i]] = lo; }   // transposed block (dX chain)
    } else img[hi_map[i]] = p;                            // biases stay fp32
}

// Stage a whole network image (weights transposed + biases, pads zero) into smem with the TMA engine.
// Called by one thread; everybody then waits on the mbarrier.
__device__ __forceinline__ void stage_weights(const NetDev &net, const float *__restrict__ img, float *sw, uint64_t *bar)
{
    fence_proxy_async();
    bulk_g2s_chunked(sw, img, (uint32_t)net.smem_w_floats * 4u, bar);
}

// Y[b][o] = act(sum_k X[b][k] * Wt[k][o] + bias[o]), b < 32.  lane -> o, warp -> 4 samples.
static __device__ void layer_forward(const float *__restrict__ X, int ldx, const float *__restrict__ Wt,
                              const float *__restrict__ bias, float *__restrict__ Y, int ldy, int in,
                              int out, bool relu)
{
    const int lane = threadIdx.x & 31, b0 = (threadIdx.x >> 5) * 4;
    const int ldw = ldw_of(out), in_pad = round_up(in, 4);
    for (int oc = 0; oc < out; oc += 64) {
        const int o0 = oc + lane, o1 = oc + lane + 32;
        const bool v0 = o0 < out, v1 = o1 < out;
        const int c0 = v0 ? o0 : 0, c1 = v1 ? o1 : 0;
        float acc[4][2];
#pragma unroll
        for (int b = 0; b < 4; ++b) { acc[b][0] = 0.f; acc[b][1] = 0.f; }
        for (int k = 0; k < in_pad; k += 4) {
            float4 x[4];
#pragma unroll
            for (int b = 0; b < 4; ++b) x[b] = *reinterpret_cast<const float4 *>(X + (b0 + b) * ldx + k);
            float w0[4], w1[4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) { w0[kk] = Wt[(k + kk) * ldw + c0]; w1[kk] = Wt[(k + kk) * ldw + c1]; }
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                acc[b][0] = fmaf(x[b].x, w0[0], acc[b][0]); acc[b][1] = fmaf(x[b].x, w1[0], acc[b][1]);
                acc[b][0] = fmaf(x[b].y, w0[1], acc[b][0]); acc[b][1] = fmaf(x[b].y, w1[1], acc[b][1]);
                acc[b][0] = fmaf(x[b].z, w0[2], acc[b][0]); acc[b][1] = fmaf(x[b].z, w1[2], acc[b][1]);
                acc[b][0] = fmaf(x[b].w, w0[3], acc[b][0]); acc[b][1] = fmaf(x[b].w, w1[3], acc[b][1]);
            }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (v0) { float y = acc[b][0] + bias[o0]; Y[(b0 + b) * ldy + o0] = (relu && y < 0.f) ? 0.f : y; }
            if (v1) { float y = acc[b][1] + bias[o1]; Y[(b0 + b) * ldy + o1] = (relu && y < 0.f) ? 0.f : y; }
        }
    }
    // the next layer reads round_up(out,4) columns with 16-byte loads: keep the pad columns zero
    const int pad = round_up(out, 4) - out;
    if (lane < pad)
#pragma unroll
        for (int b = 0; b < 4; ++b) Y[(b0 + b) * ldy + out + lane] = 0.f;
}

// dX[b][k] = (sum_o dY[b][o] * Wt[k][o]) * (Xact[b][k] > 0).  lane -> k, warp -> 4 samples.
// dY columns [out, round_up(out,4)) must be zero.
static __device__ void layer_backward_dx(const float *__restrict__ dY, int lddy, const float *__restrict__ Wt,
                                  const float *__restrict__ Xact, int ldx, float *__restrict__ dX,
                                  int lddx, int in, int out)
{
    const int lane = threadIdx.x & 31, b0 = (threadIdx.x >> 5) * 4;
    const int ldw = ldw_of(out), out4 = round_up(out, 4);
    for (int kc = 0; kc < in; kc += 64) {
        const int k0 = kc + lane, k1 = kc + lane + 32;
        const bool v0 = k0 < in, v1 = k1 < in;
        const int c0 = v0 ? k0 : 0, c1 = v1 ? k1 : 0;
        float acc[4][2];
#pragma unroll
        for (int b = 0; b < 4; ++b) { acc[b][0] = 0.f; acc[b][1] = 0.f; }
        for (int o = 0; o < out4; o += 4) {
            float4 dy[4];
#pragma unroll
            for (int b = 0; b < 4; ++b) dy[b] = *reinterpret_cast<const float4 *>(dY + (b0 + b) * lddy + o);
            float w0[4], w1[4];
#pragma unroll
            for (int oo = 0; oo < 4; ++oo) {
                const bool vo = (o + oo) < out;
                w0[oo] = vo ? Wt[c0 * ldw + o + oo] : 0.f;
                w1[oo] = vo ? Wt[c1 * ldw + o + oo] : 0.f;
            }
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                acc[b][0] = fmaf(dy[b].x, w0[0], acc[b][0]); acc[b][1] = fmaf(dy[b].x, w1[0], acc[b][1]);
                acc[b][0] = fmaf(dy[b].y, w0[1], acc[b][0]); acc[b][1] = fmaf(dy[b].y, w1[1], acc[b][1]);
                acc[b][0] = fmaf(dy[b].z, w0[2], acc[b][0]); acc[b][1] = fmaf(dy[b].z, w1[2], acc[b][1]);
                acc[b][0] = fmaf(dy[b].w, w0[3], acc[b][0]); acc[b][1] = fmaf(dy[b].w, w1[3], acc[b][1]);
            }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (v0) dX[(b0 + b) * lddx + k0] = (Xact[(b0 + b) * ldx + k0] > 0.f) ? acc[b][0] : 0.f;
            if (v1) dX[(b0 + b) * lddx + k1] = (Xact[(b0 + b) * ldx + k1] > 0.f) ? acc[b][1] : 0.f;
        }
    }
}

// gW[o][k] (+)= sum_b dY[b][o] * X[b][k];  gb[o] (+)= sum_b dY[b][o], into this CTA's partial vector.
// k = tid % 128, two 16-row groups per pass.  dY must be zero in columns [out, round_up(out,32)).
static __device__ void layer_backward_dw(const float *__restrict__ dY, int lddy, const float *__restrict__ X,
                                  int ldx, float *__restrict__ gpart, const LayerDev &L, bool accumulate)
{
    const int in = L.in, out = L.out;
    const int out_main = L.out_main;
    const int k = threadIdx.x & 127, og = threadIdx.x >> 7;
    const bool kv = k < in;
    for (int oc = 0; oc < out; oc += 32) {
        const int obase = oc + og * 16;
        float acc[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = 0.f;
        if (kv && obase < out) {
            for (int b = 0; b < kTile; ++b) {
                const float x = X[b * ldx + k];
                const float4 *dy = reinterpret_cast<const float4 *>(dY + b * lddy + obase);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 d = dy[q];
                    acc[4 * q + 0] = fmaf(d.x, x, acc[4 * q + 0]);
                    acc[4 * q + 1] = fmaf(d.y, x, acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(d.z, x, acc[4 * q + 2]);
                    acc[4 * q + 3] = fmaf(d.w, x, acc[4 * q + 3]);
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int o = obase + j;
                if (o < out) {
                    float *dst = (o < out_main) ? gpart + L.w_off + o * in + k : gpart + L.w2_off + (o - out_main) * in + k;
                    *dst = accumulate ? *dst + acc[j] : acc[j];
                }
            }
        }
    }
    for (int o = threadIdx.x; o < out; o += blockDim.x) {
        float s = 0.f;
        for (int b = 0; b < kTile; ++b) s += dY[b * lddy + o];
        float *dst = (o < out_main) ? gpart + L.b_off + o : gpart + L.b2_off + (o - out_main);
        *dst = accumulate ? *dst + s : s;
    }
}

// Full forward of one network over the 32-sample tile in plane 0.  keep_planes: trunk outputs go to
// planes 1..n (kept for backward); otherwise they ping-pong through scratch planes sA/sB.
// Raw head output (A rows + V row when dueling) lands in `head` [32][32]; then Q is formed in place.
static __device__ void net_forward(const NetDev &net, const float *sw, const float *X0, int ld0, float *smem,
                            bool keep_planes, float *sA, float *sB, float *head)
{
    const float *cur = X0; int ldc = ld0;
    const int nh = net.n_layers - 1;
    for (int l = 0; l < nh; ++l) {
        const LayerDev &L = net.L[l];
        float *dst; int ldd;
        if (keep_planes) { dst = smem + net.act_off[l + 1]; ldd = net.act_ld[l + 1]; }
        else { dst = (l & 1) ? sB : sA; ldd = kMaxDim; }
        layer_forward(cur, ldc, sw + L.smem_w, sw + L.smem_b, dst, ldd, L.in, L.out, true);
        __syncthreads();
        cur = dst; ldc = ldd;
    }
    const LayerDev &H = net.L[nh];
    layer_forward(cur, ldc, sw + H.smem_w, sw + H.smem_b, head, 32, H.in, H.out, false);
    __syncthreads();
    if (net.dueling) {                                   // Q = V + A - mean(A)   (BaseCNN.py:138)
        if (threadIdx.x < kTile) {
            float *row = head + threadIdx.x * 32;
            const int nA = net.n_actions;
            float s = 0.f;
            for (int a = 0; a < nA; ++a) s += row[a];
            const float mean = s / (float)nA, V = row[nA];
            for (int a = 0; a < nA; ++a) row[a] = V + row[a] - mean;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int argmax_row(const float *row, int n)
{
    int best = 0; float bv = row[0];
    for (int a = 1; a < n; ++a) if (row[a] > bv) { bv = row[a]; best = a; }
    return best;
}

// load 32 rows of `in` floats (row pointers in rows[]; nullptr -> zeros) into a plane, 16-byte loads
static __device__ void load_rows(const float *const *rows, float *plane, int ld, int in)
{
    const int vec = in / 4;           // in % 4 == 0 is checked on the host for the vector path
    for (int i = threadIdx.x; i < kTile * vec; i += blockDim.x) {
        const int b = i / vec, q = i - b * vec;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rows[b]) v = __ldg(reinterpret_cast<const float4 *>(rows[b]) + q);
        *reinterpret_cast<float4 *>(plane + b * ld + 4 * q) = v;
    }
    const int in_pad = round_up(in, 4);
    if (in_pad != in)
        for (int i = threadIdx.x; i < kTile * (in_pad - in); i += blockDim.x)
            plane[(i / (in_pad - in)) * ld + in + i % (in_pad - in)] = 0.f;
}

// scalar variant for in % 4 != 0
static __device__ void load_rows_scalar(const float *const *rows, float *plane, int ld, int in)
{
    const int in_pad = round_up(in, 4);
    for (int i = threadIdx.x; i < kTile * in_pad; i += blockDim.x) {
        const int b = i / in_pad, k = i - b * in_pad;
        plane[b * ld + k] = (rows[b] && k < in) ? rows[b][k] : 0.f;
    }
}


}  // namespace uavrl
