// tc_forward.cuh -- tensor-core (wgmma) forward chain of the Q-network, 3xTF32 split precision.
#pragma once
#include <vector>

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
    // loss variant of the act kernel (launch_tc_loss, federation): grid row y evaluates weight set w = loss_w0 + y on the
    // probe rows [0, S w) (loss_tri) or [S (w + 1), n) of obs = [G][S][in_dim], S = kFedProbes, with image w - loss_img0, and
    // writes loss_out[p * loss_ld + w - loss_col0] = sum over trainer p's S rows of sum_a (q_ref - Q_w)^2 / (S A), q_ref = [G][S][A]
    const float *q_ref; float *loss_out; int32_t loss_w0, loss_tri, loss_img0, loss_ld, loss_col0;
};

int tc_build(const uavrl_learner_config &c, const NetDev &net, TcNet &tc, std::vector<int32_t> &hi_map, std::vector<int32_t> &lo_map,
             std::vector<int32_t> &hi2_map, std::vector<int32_t> &lo2_map);
// tensor-core training path (tc_train.cu): forward + dX chain, then split-K dW; gradients land in l->partials
int tc_train_init(uavrl_learner *l);
// on route r = learner_route(l, B); after_chain (may be null): an event recorded after the training kernel
int launch_tc_train(uavrl_learner *l, const Route &r, const BatchSrc &src, int B, int global_batch, const float *y, int *n_grad_parts,
                    int *n_loss_parts, cudaStream_t st, cudaEvent_t after_chain);
size_t tc_smem_bytes(const TcNet &tc);
// every layer product (train: also those of the dX chain) has a compile-time wgmma chain (wgmma.cuh mma_fixed): the kernels'
// FIXED variants apply
bool tc_fixed_chains(const TcNet &tc, bool train);
// an act / TD pass over a.n rows per trainer on route r = learner_route(l, a.n)
int launch_tc_forward(uavrl_learner *l, const Route &r, const TcArgs &a, cudaStream_t st);
// the loss variant over n_weights weight sets (grid rows) on route r = learner_route(l, max_rows), max_rows = the most probe
// rows one of them evaluates
int launch_tc_loss(uavrl_learner *l, const Route &r, const TcArgs &a, int n_weights, int max_rows, cudaStream_t st);
int tc_init(uavrl_learner *l);        // builds the TC images/maps; leaves l->tc_ok = false when the net does not fit

// Stage timestamps of the tensor-core kernels (UAVRL_TC_TRACE=1, DESIGN §7): stage_trace_alloc gives a zeroed device buffer of
// kTraceSlots clock64() slots owned by m, or nullptr when tracing is off; stage_trace_print (nothing for nullptr) waits for the
// stream and prints one stderr line, the printf-formatted label then "cycles since start:" and [i]=t_i - t_0 for every written
// slot i >= 1.
constexpr int kTraceSlots = 32;
int stage_trace_alloc(DevMem &m, long long *&t);
int stage_trace_print(cudaStream_t st, const long long *t, const char *fmt, ...);

}  // namespace uavrl
