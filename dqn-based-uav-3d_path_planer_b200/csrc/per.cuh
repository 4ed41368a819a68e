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
//
// The trees belong to the replay store whose slots they index (ReplayStore::per, replay.cuh); the tree operations are
// ReplayStore members defined in per.cu.
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

// Host state of a store's trees: off unless enabled (uavrl_per_enable / uavrl_per_enable_trainers)
struct PerTree {
    PerDev dev = {};                      // the kernels' by-value argument
    uint64_t calls = 0;                   // sampling calls: the Philox counter of the draws
    DevMem mem, scratch_mem;              // owners of the trees (and wmax_bits); of the sampling scratch
    // priority of a transition stored without an error: ReplayTree.push with error 0 -> (0 + eps)^alpha, float32
    double new_priority() const { return (double)powf((float)dev.eps, (float)dev.alpha); }
};

}  // namespace uavrl
