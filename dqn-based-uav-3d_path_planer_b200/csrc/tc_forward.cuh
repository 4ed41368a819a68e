// tc_forward.cuh -- tensor-core (wgmma) forward chain of the Q-network, 3xTF32 split precision.
#pragma once
#include <vector>

#include "env.cuh"
#include "learner.cuh"

namespace uavrl {

constexpr int kTcThreads = 256;        // 2 warpgroups (m64 each); the head epilogue: warp w owns rows 32*(w%4).. (warps 0-3)
constexpr int kTcTile = 128;           // samples per CTA tile (two m64 warpgroup MMAs)

enum TcMode { kTcAct = 0, kTcArgmax = 1, kTcTdMax = 2, kTcTdGather = 3 };

struct TcArgs {
    const unsigned char *img;          // TC weight image of the network to evaluate
    int64_t img_stride;                // grouped learner (gridDim.y = G): bytes between two trainers' images; every [n] input /
                                       // output above and below is [G][n], trainer g's block at row g n
    BatchSrc src;                      // row source for the TD modes (next-state rows); unused for kTcAct
    const float *obs;                  // kTcAct: [n][in_dim]
    int32_t n, n_tiles, mode, use_next, rows_per_tile;
    float eps; int32_t is_train;
    const float *u_tape; const int32_t *rand_tape;
    uint64_t key, call;
    int32_t *actions;                  // kTcAct out / kTcArgmax out (astar) / kTcTdGather in (astar)
    float *q_out;                      // optional [n][A]
    float *y_out;                      // TD modes: y[b] = r + gamma * next_q * (1 - d)
    float gamma;
    int32_t pdl;                       // kPdlOn | kPdlEarlyWeights | kPdlEarlyRows (set by launch_tc_forward)
    long long *trace;                  // debug: CTA (0, 0) / thread 0 writes clock64() at stage boundaries (UAVRL_TC_TRACE=1)
};

int tc_build(const uavrl_learner_config &c, const NetDev &net, TcNet &tc, std::vector<int32_t> &hi_map, std::vector<int32_t> &lo_map,
             std::vector<int32_t> &hi2_map, std::vector<int32_t> &lo2_map);
// tensor-core training path (tc_train.cu): forward + dX chain, then split-K dW; gradients land in l->partials
int tc_train_init(uavrl_learner *l);
// adam != nullptr: the optimiser step may be fused behind the weight-gradient kernel (*adam_done tells whether it was)
int launch_tc_train(uavrl_learner *l, const BatchSrc &src, int B, int global_batch, const float *y, int *n_grad_parts,
                    int *n_loss_parts, cudaStream_t st, cudaEvent_t after_chain = nullptr, const AdamArgs *adam = nullptr,
                    float *loss_out = nullptr, bool *adam_done = nullptr, bool fused_td = false);
// the TD-target pass(es) can run inside the training kernel (one tile per CTA): no separate launch_tc_forward TD calls
bool tc_train_can_fuse_td(const uavrl_learner *l, int B);
// rows per tile of an act / TD pass over n samples (launch_tc_forward) and of the training kernel for a batch of B
int tc_forward_rows_per_tile(const TcNet &tc, int n);
int train_rows_per_tile(const TcNet &tc, int B);
size_t tc_smem_bytes(const TcNet &tc);
// every layer product (train: also those of the dX chain) has a compile-time wgmma chain (wgmma.cuh mma_fixed): the kernels'
// FIXED variants apply
bool tc_fixed_chains(const TcNet &tc, bool train);
// the env step fused behind the act pass (tc_forward.cu): env batch + where the step writes
struct EnvFuse { EnvDev d; float *obs_next; float *reward; uint8_t *done; };
int launch_tc_forward(uavrl_learner *l, const TcArgs &a, cudaStream_t st, const EnvFuse *fuse = nullptr);
int tc_init(uavrl_learner *l);        // builds the TC images/maps; leaves l->tc_ok = false when the net does not fit

}  // namespace uavrl
