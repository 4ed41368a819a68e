// per.cuh -- prioritised experience replay on the device (SURVEY.md 8f-3).
//
// Reference: BaseClass/replay_buffer.py:57-223 -- SumTree (array heap, 2*capacity-1 nodes) + ReplayTree (alpha 0.6,
// beta 0.4 -> 1 by 0.001 per sampling call, epsilon 0.01, error clip 1, stratified sampling over `batch` equal
// segments of int(total), importance weights (n * p / total)^-beta normalised by their maximum).
//
// GPU form.  SumTree.get_leaf(v) returns the first leaf, in the heap's left-to-right leaf order, whose inclusive
// prefix sum reaches v.  That order is the data order rotated by rot = 2^ceil(log2 cap) - cap (the leaves of the
// deepest heap level come first), so the heap is replaced by three flat fp64 levels over *positions*
// j = (slot - rot) mod cap:   leaf[cap] (stored by slot), l1 = sums of 32 positions, l2 = sums of 32 l1 entries.
// Sampling: every CTA scans l2 in shared memory, then one warp per sample does two 32-wide scans (l1 group, leaves).
// Updating B priorities: three small launches (leaves, touched l1 entries, touched l2 entries), each entry recomputed
// from its 32 children in a fixed order -> deterministic, no atomics, duplicates idempotent.  The sums differ from the
// reference's incrementally updated heap nodes only in fp64 rounding (~1e-16 relative).
//
// Grouped learner (uavrl_per_enable_trainers): one tree per trainer, as every reference Trainer owns its replay.  Trainer g's
// tree covers its own transitions under trainer-local slots j = f Ng + (e - g Ng) (ring frame f, env e of block g), which is
// how a stand-alone learner over Ng envs numbers its slots.  Every array is [G][...] (leaf [G][cap], l1 [G][n1], l2 [G][n2],
// scratch [G][B], wmax_bits [G]) and every kernel takes the trainer from blockIdx.y; cap, rot, alpha, beta and the sampling
// call counter are shared (the trainers sample in lockstep).  G = 1 is the single tree above.
#pragma once
#include <math.h>

#include "common.cuh"

namespace uavrl {

constexpr int kPerMaxL2 = 4096;          // l2 entries scanned in shared memory: capacity <= 4096 * 1024 slots (per trainer)

struct PerDev {
    int32_t enabled;
    int32_t G;                            // trees (one per trainer)
    int64_t cap, rot, n1, n2;             // per tree
    double *leaf, *l1, *l2;
    double alpha, beta, beta_inc, eps, err_upper;
    // scratch of the integrated update path, [G][scratch_cap] (wmax_bits [G])
    int32_t *idx; float *w, *abs_err; double *w_raw; unsigned long long *wmax_bits;
    int32_t scratch_cap;
};

}  // namespace uavrl

struct uavrl_learner;
namespace uavrl {
// Every call below acts on each trainer's tree at once (grid y = G): per_fill_range fills the same trainer-local range in
// every tree; per_set takes [G][n] slots / values; per_sample draws B per trainer into [G][B] outputs (u_tape [G][B]).
// contiguous slots (mod cap): the first n_first get `value`, the rest `value_rest` (n_first < 0: all get `value`)
int per_fill_range(uavrl_learner *l, int64_t first_slot, int64_t n, double value, cudaStream_t st, int64_t n_first = -1,
                   double value_rest = 0.0);
// priority of a transition stored without an error: ReplayTree.push with error 0 -> (0 + eps)^alpha, float32
inline double per_new_priority(const PerDev &p) { return (double)powf((float)p.eps, (float)p.alpha); }
int per_sample(uavrl_learner *l, int B, const double *u_tape, int32_t *slot_out, float *w_out, cudaStream_t st);
int per_set(uavrl_learner *l, int n, const int32_t *slots, const double *prio, const float *abs_err, int clip, cudaStream_t st);
}  // namespace uavrl
