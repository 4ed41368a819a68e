// federate.cu -- selective federated aggregation across the trainers of a grouped learner, sm_90a.
//
// Replaces Envs/PathPlan_City.py:644-684 (Federated_Learning_choice), the reference's aggregation for DQN-family trainers.
// Round p = 0 .. G-1, in this order and in place:
//   1. probe states: 10 distinct transitions of trainer p's own replay (random.sample), their state rows;
//   2. q_value = Q_p(probes) with trainer p's parameters as they stand (they change only in round p);
//   3. loss_q = mse(q_value, Q_q(probes)) for every q != p with trainer q's CURRENT parameters (already replaced for q < p);
//   4. the stable sort by loss (equal losses keep ascending q), the first k = (G - 1) / 2;
//   5. theta_p <- (theta_p + theta_c0 + theta_c1 + ...) / (k + 1): float32, left to right, one division;
//   6. only q_local is written (replace_param); q_target, the Adam moments and the counters stay.
//
// Schedule (every launch on the caller's stream, no host synchronisation):
//   probe rows (ring: one gather kernel)          -> probes [G][10][in]
//   the act pass on the probes                    -> q_ref [G][10][A]          (block g of rows -> trainer g)
//   loss variant of the act pass, G weight sets   -> M[p][q], q > p, initial parameters (stay valid until round p)
//   per round p: rank (M row p) -> average -> refresh trainer p's fp32 / tensor-core images -> loss variant with the new
//                theta_p on the probes of every p' > p -> column p of M
// so the forwards evaluate G (G - 1) 10 rows in all, and a call makes 5 G + 2 kernel launches (4 G + 2 without tensor cores;
// one fewer with explicit probe states) plus three memsets.
//
// Sharded form (uavrl_learner_fed_shard): W learners of G_local trainers each hold the global trainers [r G_local, (r + 1) G_local)
// of G = G_local W.  Three calls with two all-gathers between them, made by the caller:
//   local    probe rows and the act pass of the own trainers -> [probes | q_ref | q_local] rows of x0        -> gather x0
//   columns  M[p][q], q in the own slice, p < q: the own (initial) images on the gathered probes -> x1 slice -> gather x1
//   rounds   every rank runs every round on identical inputs, averaging into a flat replica of all G q_local vectors and
//            repacking one scratch image of theta_p per round; at the end the own slice goes back to q_local.
// Every M entry is one tile's fixed-order sum on the route the global probe-row count picks, so the rounds see the losses the
// one-GPU call computes, and the result is that call's, bit for bit.  The column phase keeps contiguous slices: rank r evaluates
// S (q - 1) rows for each of its q, so the last rank does the most, about (2W - 1) / W^2 of the pass.
#include "learner.cuh"
#include "mlp_tile.cuh"
#include "tc_forward.cuh"

#include <string.h>

#include <string>

namespace uavrl {

// probe states of every trainer from the lockstep ring: 10 distinct trainer-local logical indices (perm_index keyed by
// seed + g and the call counter, or row g of a [G][10] tape), their state rows copied to probes[g]
__global__ void fed_probe_kernel(BatchSrc src, int in_dim, uint64_t fed_key, uint64_t call, float *__restrict__ probes,
                                 int32_t *__restrict__ idx_out)
{
    __shared__ const float *rows[kFedProbes];
    const int g = blockIdx.x;
    if (threadIdx.x < kFedProbes) {
        BatchSrc sg = trainer_src(src, g, kFedProbes, in_dim);
        sg.key = trainer_key(fed_key, kFedSalt, g);
        uint32_t pkey[4];
        Philox::gen(sg.key, call, 0xFEDull, pkey);
        const int s = threadIdx.x;
        const int64_t j = sg.idx_tape ? (int64_t)sg.idx_tape[s] : (int64_t)perm_index((uint64_t)s, (uint64_t)sg.count, pkey);
        const float *sp, *s2p;
        resolve_rows(sg, s, in_dim, pkey, sp, s2p);
        rows[s] = sp;
        if (idx_out) idx_out[(size_t)g * kFedProbes + s] = (int32_t)j;
    }
    __syncthreads();
    float *out = probes + (size_t)g * kFedProbes * in_dim;
    for (int i = threadIdx.x; i < kFedProbes * in_dim; i += blockDim.x) out[i] = rows[i / in_dim][i % in_dim];
}

// loss -> an unsigned key with the order of the floats (NaN last)
__device__ __forceinline__ uint32_t loss_key(float x)
{
    const uint32_t u = __float_as_uint(x);
    if (x != x) return 0xFFFFFFFFu;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// round p's selection: candidate q's rank among q' != p under (loss, index); rank < k -> chosen[p][rank] = q.  One thread per
// candidate over any number of CTAs; row p of M is staged through shared memory in chunks.
constexpr int kRankChunk = 2048;
__global__ void __launch_bounds__(256) fed_rank_kernel(int G, int p, int k, int kk, const float *__restrict__ M, int32_t *__restrict__ chosen)
{
    __shared__ uint32_t keys[kRankChunk];
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const float *row = M + (size_t)p * G;
    const uint32_t kq = q < G ? loss_key(row[q]) : 0u;
    int rank = 0;
    for (int c0 = 0; c0 < G; c0 += kRankChunk) {
        const int n = G - c0 < kRankChunk ? G - c0 : kRankChunk;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = loss_key(row[c0 + i]);
        __syncthreads();
        if (q < G && q != p)
            for (int i = 0; i < n; ++i) {
                const int q2 = c0 + i;
                const uint32_t k2 = keys[i];
                rank += (q2 != p) && (k2 < kq || (k2 == kq && q2 < q));
            }
    }
    if (q < G && q != p && rank < k) chosen[(size_t)p * kk + rank] = q;
}

// theta_p <- (theta_p + theta_c0 + ... + theta_c{k-1}) / (k + 1): every addition and the division individually rounded (no FMA
// contraction, no reassociation); the loads of 8 chosen rows are issued ahead of their additions
__global__ void __launch_bounds__(256) fed_average_kernel(int P, int p, int k, const int32_t *__restrict__ chosen, float *__restrict__ local)
{
    __shared__ int32_t c[256];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float s = i < P ? local[(size_t)p * P + i] : 0.f;
    for (int j0 = 0; j0 < k; j0 += 256) {
        const int n = k - j0 < 256 ? k - j0 : 256;
        __syncthreads();
        if ((int)threadIdx.x < n) c[threadIdx.x] = chosen[j0 + threadIdx.x];
        __syncthreads();
        if (i < P) {
            int j = 0;
            for (; j + 8 <= n; j += 8) {
                float v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = local[(size_t)c[j + u] * P + i];
#pragma unroll
                for (int u = 0; u < 8; ++u) s = __fadd_rn(s, v[u]);
            }
            for (; j < n; ++j) s = __fadd_rn(s, local[(size_t)c[j] * P + i]);
        }
    }
    if (i < P) local[(size_t)p * P + i] = __fdiv_rn(s, (float)(k + 1));
}

// ---- the sharded form
static size_t fed_seg(const uavrl_learner *l) { return (size_t)kFedProbes * (l->net.in_dim + l->net.n_actions) + l->net.P; }

// rows x width floats between two pitched device arrays (pitches in floats)
static int copy_rows(float *dst, size_t dpitch, const float *src, size_t spitch, size_t width, size_t rows, cudaStream_t st)
{
    UAVRL_CUDA(cudaMemcpy2DAsync(dst, dpitch * 4, src, spitch * 4, width * 4, rows, cudaMemcpyDeviceToDevice, st));
    return 0;
}

static int fed_declared(const uavrl_learner *l, const char *fn)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (!l->fed.world) return fail(UAVRL_ERR_STATE, std::string(fn) + " before uavrl_learner_fed_shard");
    return 0;
}

static int fed_phase_is(const uavrl_learner *l, int phase, const char *fn)
{
    if (int rc = fed_declared(l, fn)) return rc;
    static const char *want[3] = { "", "after uavrl_learner_fed_local and the gather of exchange 0",
                                   "after uavrl_learner_fed_columns and the gather of exchange 1" };
    if (l->fed.phase != phase) return fail(UAVRL_ERR_STATE, std::string(fn) + " called out of order: it runs " + want[phase]);
    return 0;
}

}  // namespace uavrl

using namespace uavrl;

extern "C" {

int uavrl_learner_federate(uavrl_learner *l, const float *probe_states_dev, const int32_t *probe_tape_dev, int32_t *probe_idx_out_dev,
                           float *loss_out_dev, int32_t *chosen_out_dev, void *stream)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (probe_states_dev && probe_tape_dev)
        return fail(UAVRL_ERR_INVALID, "uavrl_learner_federate: give probe states or a probe tape, not both");
    const int G = l->G;
    if (G == 1) return 0;
    const bool ring = probe_states_dev == nullptr;
    if (ring && (l->replay.mode != kReplayLockstep || l->replay.count / G < kFedProbes))
        return fail(UAVRL_ERR_INVALID, "uavrl_learner_federate: every trainer needs at least 10 transitions in the ring to draw probe states from");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int k = (G - 1) / 2, kk = k > 0 ? k : 1, in = l->net.in_dim, A = l->net.n_actions, P = l->net.P;
    const size_t rows = (size_t)G * kFedProbes;
    // per-call scratch, stream-ordered
    float *probes = nullptr, *q_ref = nullptr, *M = loss_out_dev;
    int32_t *acts = nullptr, *chosen = chosen_out_dev;
    bool ok = true;
    auto alloc = [&](void **p, size_t bytes) { if (ok && cudaMallocAsync(p, bytes, st) != cudaSuccess) ok = false; };
    if (ring) alloc((void **)&probes, rows * in * 4);
    alloc((void **)&q_ref, rows * A * 4);
    alloc((void **)&acts, rows * 4);
    if (!M) alloc((void **)&M, (size_t)G * G * 4);
    if (!chosen) alloc((void **)&chosen, (size_t)G * kk * 4);
    int rc = 0;
    auto done = [&](int code) {
        if (probes) cudaFreeAsync(probes, st);
        if (q_ref) cudaFreeAsync(q_ref, st);
        if (acts) cudaFreeAsync(acts, st);
        if (M && M != loss_out_dev) cudaFreeAsync(M, st);
        if (chosen && chosen != chosen_out_dev) cudaFreeAsync(chosen, st);
        return code;
    };
    if (!ok) { cudaGetLastError(); return done(fail(UAVRL_ERR_CUDA, "uavrl_learner_federate: out of device memory for the scratch")); }
    // 1. probe rows
    if (ring) {
        BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, probe_tape_dev);
        fed_probe_kernel<<<G, 256, 0, st>>>(src, in, l->cfg.seed ^ kFedSalt, l->fed_calls++, probes, probe_idx_out_dev);
        UAVRL_LAUNCHED();
    } else if (probe_idx_out_dev) {
        if (cudaMemsetAsync(probe_idx_out_dev, 0xFF, rows * 4, st) != cudaSuccess)             // no replay indices: -1
            return done(fail(UAVRL_ERR_CUDA, "uavrl_learner_federate: cudaMemsetAsync failed"));
    }
    const float *pr = ring ? probes : probe_states_dev;
    // 2. own Q of every trainer on its probes: the grouped act pass (greedy; not an act call, so its Philox counter stays)
    const uint64_t calls = l->act_calls;
    if ((rc = launch_act(l, pr, (int)rows, 0.f, 0, nullptr, nullptr, acts, q_ref, st))) return done(rc);
    l->act_calls = calls;
    // 3. losses of the initial parameters: M[p][q], q > p; [p][p] = 0
    if (cudaMemsetAsync(M, 0, (size_t)G * G * 4, st) != cudaSuccess || cudaMemsetAsync(chosen, 0xFF, (size_t)G * kk * 4, st) != cudaSuccess)
        return done(fail(UAVRL_ERR_CUDA, "uavrl_learner_federate: cudaMemsetAsync failed"));
    const FedLoss fl = { pr, q_ref, M, G, G, 0, 0, l->img_local, l->tc_img_local };
    if ((rc = launch_fed_loss(l, fl, 0, G, true, st))) return done(rc);
    if (k == 0) {                                                    // G = 2: nothing is averaged, M[1][0] from the same parameters
        if ((rc = launch_fed_loss(l, fl, 0, G, false, st))) return done(rc);
        return done(0);
    }
    const int tf = l->tc.train_img_bytes / 4, wf = l->net.smem_w_floats;
    const int pb = (P + 255) / 256;
    for (int p = 0; p < G; ++p) {
        fed_rank_kernel<<<(G + 255) / 256, 256, 0, st>>>(G, p, k, kk, M, chosen);
        UAVRL_LAUNCHED();
        fed_average_kernel<<<pb, 256, 0, st>>>(P, p, k, chosen + (size_t)p * kk, l->local);
        UAVRL_LAUNCHED();
        // trainer p's kernel-layout images of q_local (the target images are not touched)
        pack_image_kernel<<<pb, 256, 0, st>>>(P, l->local + (size_t)p * P, l->img_map, l->img_local + (size_t)p * wf, wf);
        UAVRL_LAUNCHED();
        if (l->tc_ok) {
            pack_tc_kernel<<<pb, 256, 0, st>>>(P, l->local + (size_t)p * P, l->tc_hi_map, l->tc_lo_map, l->tc_hi2_map, l->tc_lo2_map,
                                               (float *)l->tc_img_local + (size_t)p * tf, tf);
            UAVRL_LAUNCHED();
        }
        // the new theta_p on the probes of every later round: column p of M
        if (p + 1 < G && (rc = launch_fed_loss(l, fl, p, 1, false, st))) return done(rc);
    }
    l->chain.launched(kChainNone);
    return done(0);
}

int uavrl_learner_fed_shard(uavrl_learner *l, int32_t rank, int32_t world)
{
    if (!l) return fail(UAVRL_ERR_INVALID, "null learner");
    if (world < 1 || rank < 0 || rank >= world) return fail(UAVRL_ERR_INVALID, "uavrl_learner_fed_shard: needs world >= 1 and rank in [0, world)");
    const int64_t G = (int64_t)l->G * world;
    if (G > 65535) return fail(UAVRL_ERR_INVALID, "uavrl_learner_fed_shard: the global trainer count (trainers x world) must be at most 65535");
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    const size_t Gs = (size_t)G, GL = (size_t)l->G, S = kFedProbes, in = l->net.in_dim, A = l->net.n_actions, P = l->net.P;
    const size_t k = (Gs - 1) / 2, kk = k > 0 ? k : 1;
    FedShard f;                                                  // built beside the current state, swapped in when complete
    f.rank = rank; f.world = world;
    int rc;
    if ((rc = f.mem.alloc(f.x0, Gs * fed_seg(l), false)) || (rc = f.mem.alloc(f.x1, Gs * Gs, false)) ||
        (rc = f.mem.alloc(f.probes, Gs * S * in, false)) || (rc = f.mem.alloc(f.q_ref, Gs * S * A, false)) ||
        (rc = f.mem.alloc(f.rep, Gs * P, false)) || (rc = f.mem.alloc(f.M, Gs * Gs, false)) || (rc = f.mem.alloc(f.chosen, Gs * kk, false)) ||
        (rc = f.mem.alloc(f.l_probes, GL * S * in, false)) || (rc = f.mem.alloc(f.l_q, GL * S * A, false)) ||
        (rc = f.mem.alloc(f.acts, GL * S, false)) ||
        (rc = f.mem.alloc(f.img, (size_t)l->net.smem_w_floats)))  // zeroed: the pads of a packed image stay 0
        return rc;
    if (l->tc_ok && (rc = f.mem.alloc(f.tc_img, (size_t)l->tc.train_img_bytes))) return rc;
    l->fed = std::move(f);
    return 0;
}

float *uavrl_learner_fed_exchange_ptr(uavrl_learner *l, int32_t phase, int64_t *len_out)
{
    if (!l || !l->fed.world || (phase != 0 && phase != 1)) return nullptr;
    const int64_t G = (int64_t)l->G * l->fed.world;
    if (len_out) *len_out = phase == 0 ? G * (int64_t)fed_seg(l) : G * G;
    return phase == 0 ? l->fed.x0 : l->fed.x1;
}

int uavrl_learner_fed_local(uavrl_learner *l, const float *probe_states_dev, const int32_t *probe_tape_dev, int32_t *probe_idx_out_dev,
                            void *stream)
{
    if (int rc = fed_declared(l, "uavrl_learner_fed_local")) return rc;
    if (probe_states_dev && probe_tape_dev)
        return fail(UAVRL_ERR_INVALID, "uavrl_learner_fed_local: give probe states or a probe tape, not both");
    FedShard &f = l->fed;
    const int GL = l->G, G = GL * f.world;
    const bool ring = probe_states_dev == nullptr;
    if (G > 1 && ring && (l->replay.mode != kReplayLockstep || l->replay.count / GL < kFedProbes))
        return fail(UAVRL_ERR_INVALID, "uavrl_learner_fed_local: every trainer needs at least 10 transitions in the ring to draw probe states from");
    if (G > 1) {
        UAVRL_CUDA(cudaSetDevice(l->cfg.device));
        const cudaStream_t st = (cudaStream_t)stream;
        const size_t S = kFedProbes, in = l->net.in_dim, A = l->net.n_actions, P = l->net.P, seg = fed_seg(l);
        if (ring) {
            BatchSrc src = l->replay.source(l->cfg.seed, l->epoch, probe_tape_dev);
            fed_probe_kernel<<<GL, 256, 0, st>>>(src, (int)in, l->cfg.seed ^ kFedSalt, l->fed_calls++, f.l_probes, probe_idx_out_dev);
            UAVRL_LAUNCHED();
        } else if (probe_idx_out_dev) {
            UAVRL_CUDA(cudaMemsetAsync(probe_idx_out_dev, 0xFF, (size_t)GL * S * 4, st));          // no replay indices: -1
        }
        const float *pr = ring ? f.l_probes : probe_states_dev;
        const uint64_t calls = l->act_calls;                    // not an act call: its Philox counter stays
        const int rc = launch_act(l, pr, GL * kFedProbes, 0.f, 0, nullptr, nullptr, f.acts, f.l_q, st);
        l->act_calls = calls;
        if (rc) return rc;
        float *mine = f.x0 + (size_t)f.rank * GL * seg;
        if (int e = copy_rows(mine, seg, pr, S * in, S * in, GL, st)) return e;
        if (int e = copy_rows(mine + S * in, seg, f.l_q, S * A, S * A, GL, st)) return e;
        if (int e = copy_rows(mine + S * (in + A), seg, l->local, P, P, GL, st)) return e;
        l->chain.launched(kChainNone);
    }
    f.phase = 1;
    return 0;
}

int uavrl_learner_fed_columns(uavrl_learner *l, void *stream)
{
    if (int rc = fed_phase_is(l, 1, "uavrl_learner_fed_columns")) return rc;
    FedShard &f = l->fed;
    const int GL = l->G, G = GL * f.world;
    if (G > 1) {
        UAVRL_CUDA(cudaSetDevice(l->cfg.device));
        const cudaStream_t st = (cudaStream_t)stream;
        const size_t S = kFedProbes, in = l->net.in_dim, A = l->net.n_actions, P = l->net.P, seg = fed_seg(l);
        int rc;
        if ((rc = copy_rows(f.probes, S * in, f.x0, seg, S * in, G, st)) || (rc = copy_rows(f.q_ref, S * A, f.x0 + S * in, seg, S * A, G, st)) ||
            (rc = copy_rows(f.rep, P, f.x0 + S * (in + A), seg, P, G, st)))
            return rc;
        float *cols = f.x1 + (size_t)f.rank * G * GL;                // [G][G_local]: column q of M at q - rank G_local; [q][q] = 0
        UAVRL_CUDA(cudaMemsetAsync(cols, 0, (size_t)G * GL * 4, st));
        const int c0 = f.rank * GL;
        const FedLoss fl = { f.probes, f.q_ref, cols, G, GL, c0, c0, l->img_local, l->tc_img_local };
        if ((rc = launch_fed_loss(l, fl, c0, GL, true, st))) return rc;
        if ((G - 1) / 2 == 0 && (rc = launch_fed_loss(l, fl, c0, GL, false, st))) return rc;   // G = 2: the whole column
    }
    f.phase = 2;
    return 0;
}

int uavrl_learner_fed_rounds(uavrl_learner *l, float *loss_out_dev, int32_t *chosen_out_dev, void *stream)
{
    if (int rc = fed_phase_is(l, 2, "uavrl_learner_fed_rounds")) return rc;
    FedShard &f = l->fed;
    const int GL = l->G, W = f.world, G = GL * W;
    if (G == 1) { f.phase = 0; return 0; }
    UAVRL_CUDA(cudaSetDevice(l->cfg.device));
    const cudaStream_t st = (cudaStream_t)stream;
    const int k = (G - 1) / 2, kk = k > 0 ? k : 1, P = l->net.P;
    float *M = loss_out_dev ? loss_out_dev : f.M;
    int32_t *chosen = chosen_out_dev ? chosen_out_dev : f.chosen;
    int rc;
    for (int r = 0; r < W; ++r)                                      // rank r's columns [G][G_local] into M [G][G]
        if ((rc = copy_rows(M + (size_t)r * GL, G, f.x1 + (size_t)r * G * GL, GL, GL, G, st))) return rc;
    UAVRL_CUDA(cudaMemsetAsync(chosen, 0xFF, (size_t)G * kk * 4, st));
    if (k > 0) {
        const int tf = l->tc.train_img_bytes / 4, wf = l->net.smem_w_floats, pb = (P + 255) / 256;
        for (int p = 0; p < G; ++p) {
            fed_rank_kernel<<<(G + 255) / 256, 256, 0, st>>>(G, p, k, kk, M, chosen);
            UAVRL_LAUNCHED();
            fed_average_kernel<<<pb, 256, 0, st>>>(P, p, k, chosen + (size_t)p * kk, f.rep);
            UAVRL_LAUNCHED();
            if (p + 1 == G) break;
            // theta_p's images in the scratch, then column p of M
            pack_image_kernel<<<pb, 256, 0, st>>>(P, f.rep + (size_t)p * P, l->img_map, f.img, wf);
            UAVRL_LAUNCHED();
            if (l->tc_ok) {
                pack_tc_kernel<<<pb, 256, 0, st>>>(P, f.rep + (size_t)p * P, l->tc_hi_map, l->tc_lo_map, l->tc_hi2_map, l->tc_lo2_map,
                                                   (float *)f.tc_img, tf);
                UAVRL_LAUNCHED();
            }
            const FedLoss fl = { f.probes, f.q_ref, M, G, G, 0, p, f.img, f.tc_img };
            if ((rc = launch_fed_loss(l, fl, p, 1, false, st))) return rc;
        }
        // the own trainers: their averaged q_local and its kernel-layout images (the target images are not touched)
        UAVRL_CUDA(cudaMemcpyAsync(l->local, f.rep + (size_t)f.rank * GL * P, (size_t)GL * P * 4, cudaMemcpyDeviceToDevice, st));
        const dim3 blocks(pb, GL);
        pack_image_kernel<<<blocks, 256, 0, st>>>(P, l->local, l->img_map, l->img_local, wf);
        UAVRL_LAUNCHED();
        if (l->tc_ok) {
            pack_tc_kernel<<<blocks, 256, 0, st>>>(P, l->local, l->tc_hi_map, l->tc_lo_map, l->tc_hi2_map, l->tc_lo2_map,
                                                   (float *)l->tc_img_local, tf);
            UAVRL_LAUNCHED();
        }
    }
    l->chain.launched(kChainNone);
    f.phase = 0;
    return 0;
}

}  // extern "C"
