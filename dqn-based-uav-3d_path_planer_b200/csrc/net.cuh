// net.cuh -- what the Q-network and SAC learners share about their networks and trainer groups: the fp32 MLP description the
// SMEM-resident kernels follow (mlp_tile.cuh) and the create-time rules of a learner holding G trainers.
#pragma once
#include "common.cuh"

namespace uavrl {

constexpr int kTile = 32;             // samples per CTA tile
constexpr int kNetThreads = 256;      // 8 warps: lane -> output unit, warp -> 4 samples
constexpr int kMaxDim = 128;          // every layer width (and in_dim) <= 128
constexpr int kMaxLayers = UAVRL_MAX_HIDDEN + 1;   // trunk layers + (combined) head

__host__ __device__ inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// One dense layer as the kernels see it.  Weights live in smem transposed: Wt[k][o], ld = out+1
// (odd when out is even -> conflict-free whether lanes walk o or k).
struct LayerDev {
    int32_t in, out;                  // out of the head = n_actions (+1 value row when dueling)
    int32_t w_off, b_off;             // offsets in the flat state_dict-ordered parameter vector
    int32_t w2_off, b2_off;           // second head block (rows out_main..out-1): dueling fc_V, SAC actor fc_std; -1 if none
    int32_t out_main;                 // rows served by (w_off, b_off)
    int32_t smem_w, smem_b;           // offsets (floats) inside the smem weight area
};

struct NetDev {
    int32_t in_dim, n_layers, n_actions, dueling;
    int32_t P;                        // parameter count
    int32_t smem_w_floats;            // total smem floats for Wt + biases
    int32_t act_off[kMaxLayers + 1];  // smem offsets of the activation planes X0, H1.. (floats)
    int32_t act_ld[kMaxLayers + 1];
    int32_t smem_total_floats;        // whole dynamic smem carve-up for the update kernel
    LayerDev L[kMaxLayers];
};

// generic MLP description: trunk widths + head = `head_main` rows (+ `head_extra` rows from a second parameter block)
inline int build_mlp(int in_dim, int n_hidden, const int32_t *hidden, int head_main, int head_extra, NetDev &n)
{
    memset(&n, 0, sizeof(n));
    if (in_dim <= 0 || in_dim > kMaxDim) return fail(UAVRL_ERR_INVALID, "in_dim must be in [1,128]");
    if (n_hidden < 1 || n_hidden > UAVRL_MAX_HIDDEN) return fail(UAVRL_ERR_INVALID, "n_hidden must be in [1,4]");
    if (head_main < 1 || head_main + head_extra > 32) return fail(UAVRL_ERR_INVALID, "head width must be in [1,32]");
    n.in_dim = in_dim; n.n_actions = head_main; n.dueling = 0;
    n.n_layers = n_hidden + 1;
    int in = in_dim, poff = 0, soff = 0;
    for (int l = 0; l < n.n_layers; ++l) {
        LayerDev &L = n.L[l];
        const bool head = (l == n_hidden);
        const int out_real = head ? head_main : hidden[l];
        if (out_real <= 0 || out_real > kMaxDim) return fail(UAVRL_ERR_INVALID, "hidden width must be in [1,128]");
        L.in = in;
        L.out = out_real + (head ? head_extra : 0);
        L.out_main = out_real;
        L.w_off = poff; poff += out_real * in;
        L.b_off = poff; poff += out_real;
        L.w2_off = L.b2_off = -1;
        if (head && head_extra > 0) { L.w2_off = poff; poff += head_extra * in; L.b2_off = poff; poff += head_extra; }
        const int ldw = (L.out % 2 == 0) ? L.out + 1 : L.out;
        L.smem_w = soff; soff += round_up(in, 4) * ldw;
        L.smem_b = soff; soff += round_up(L.out, 4);
        in = out_real;
    }
    n.P = poff;
    n.smem_w_floats = round_up(soff, 4);
    int off = n.smem_w_floats;
    // activation planes: X0 (input), H1..Hn (trunk outputs); ld = round_up(dim,32)
    for (int i = 0; i <= n_hidden; ++i) {
        const int dim = (i == 0) ? in_dim : hidden[i - 1];
        n.act_ld[i] = round_up(dim, 32);
        n.act_off[i] = off; off += kTile * n.act_ld[i];
    }
    n.smem_total_floats = off;   // kernels append their own extra planes after this
    return 0;
}

// The refusals both trainer-group create entry points make (uavrl_learner_create_trainers, uavrl_sac_create_trainers) after the
// learner's own configuration checks and before anything is allocated; on success cfg.device is current.  `learner` names the
// handle in the no-device message.
template <class Config>
int check_trainer_group(const Config &cfg, int32_t n_trainers, const char *learner)
{
    if (n_trainers < 1 || n_trainers > 65535)        // every grouped kernel runs one grid row per trainer: gridDim.y <= 65535
        return fail(UAVRL_ERR_INVALID, "n_trainers must be in [1, 65535]");
    if (n_trainers > 1 && (cfg.lockstep_envs < 0 || cfg.lockstep_envs % n_trainers != 0))
        return fail(UAVRL_ERR_INVALID, "lockstep_envs must be a multiple of n_trainers (every trainer owns lockstep_envs / n_trainers envs)");
    if (n_trainers > 1 && cfg.replay_capacity / n_trainers <= 0)
        return fail(UAVRL_ERR_INVALID, "replay_capacity / n_trainers must be > 0");
    if (cfg.batch_size <= 0 || cfg.replay_capacity <= 0) return fail(UAVRL_ERR_INVALID, "batch_size and replay_capacity must be > 0");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(UAVRL_ERR_CUDA, std::string("no CUDA device: the ") + learner + " has no CPU fallback");
    UAVRL_CUDA(cudaSetDevice(cfg.device));
    return 0;
}

// Gradient / loss partial slots per trainer: a single trainer keeps max_ctas (any batch); a grouped learner sizes them from its
// per-trainer batch (the grid of its widest update kernel) and grows them when a larger explicit batch arrives.
inline int32_t trainer_parts_cap(int32_t G, int32_t batch_size, int32_t max_ctas)
{
    const int32_t tiles = (batch_size + kTile - 1) / kTile;
    return (G == 1 || tiles > max_ctas) ? max_ctas : tiles;
}

// Entry points a learner of G > 1 trainers does not offer (`what` names the call): refused before anything is enqueued or
// allocated.
inline int refuse_grouped(int G, const std::string &what)
{
    if (G > 1) return fail(UAVRL_ERR_INVALID, what + " is not available on a learner with " + std::to_string(G) + " trainers");
    return 0;
}

}  // namespace uavrl
