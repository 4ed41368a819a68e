// launch_chain.cuh -- which kernel of a Q-network learner's stream launches with programmatic dependent launch (PDL, see
// common.cuh), and what its prologue may fetch before griddepcontrol.wait.  A wrong early fetch is a data race, so every
// such decision is taken here, from the kind of kernel launched last.  Host only: tests/test_launch_chain_cpu.py compiles it
// with g++ and checks every rule.
#pragma once
#include <atomic>

namespace uavrl {

extern std::atomic<int> g_pdl;            // uavrl_set_pdl(); default on

// TcArgs.pdl / kernel flags
constexpr int kPdlOn = 1, kPdlEarlyWeights = 2, kPdlEarlyRows = 4;

// The kernels of the chain.  kChainNone is every other kernel (the fp32 act and update kernels, prioritised replay,
// federation, apply_grads): it launches plainly, and the kernel after it does not overlap it.
enum ChainKernel {
    kChainNone = 0,
    kChainAct,           // tensor-core act
    kChainEnv,           // env step of the Q-network loops
    kChainTd,            // tensor-core TD-target pass
    kChainTrain,         // tensor-core training kernel behind separate TD passes
    kChainTrainFusedTd,  // tensor-core training kernel that forms the TD targets itself
    kChainDw,            // weight-gradient kernel
    kChainAdam,          // reduce + Adam, all-reduce + Adam
};

struct ChainLaunch {
    bool pdl;            // launch with PDL: the prologue overlaps the predecessor's tail
    bool early_weights;  // the weight image may be staged before the wait: the predecessor does not write it
    bool early_rows;     // the first tile's rows may be gathered before the wait: the predecessor does not write them
    int flags() const { return pdl ? kPdlOn | (early_weights ? kPdlEarlyWeights : 0) | (early_rows ? kPdlEarlyRows : 0) : 0; }
};

// How kernel k launches behind prev.  on: inside a ChainScope with uavrl_set_pdl(1); off, everything launches plainly.
inline ChainLaunch chain_launch(ChainKernel k, ChainKernel prev, bool on)
{
    ChainLaunch c = { false, false, false };
    if (!on) return c;
    switch (k) {
    case kChainAct:
        c.pdl = prev != kChainNone;
        c.early_rows = prev == kChainAdam;      // obs frame written by the env step two kernels back, weights by Adam
        c.early_weights = prev == kChainEnv;    // collection-only iteration: weights untouched, obs just written
        break;
    case kChainTd:
        c.pdl = prev != kChainNone;
        c.early_weights = prev == kChainEnv || prev == kChainTd;   // neither the env step nor a TD pass writes weight images
        break;
    case kChainEnv: c.pdl = prev == kChainAct; break;
    case kChainTrain: c.pdl = prev == kChainTd; break;
    case kChainTrainFusedTd: c.pdl = prev == kChainEnv; break;
    case kChainDw: c.pdl = true; break;
    case kChainAdam: c.pdl = prev == kChainDw; break;
    case kChainNone: break;
    }
    return c;
}

// The chain state of one learner's stream: ask next() before a launch, call launched() after it.
class LaunchChain {
public:
    ChainLaunch next(ChainKernel k) const { return chain_launch(k, prev_, on()); }
    void launched(ChainKernel k) { prev_ = scoped_ ? k : kChainNone; }

private:
    friend class ChainScope;
    bool on() const { return scoped_ && g_pdl.load() != 0; }
    bool scoped_ = false;
    ChainKernel prev_ = kChainNone;
};

// Turns the chain on for the kernels launched while it lives.  The first of them launches plainly: whatever precedes it on
// the stream is not the chain's.  A scope opened inside another changes nothing.
class ChainScope {
public:
    explicit ChainScope(LaunchChain &c) : c_(c), outer_(c.scoped_)
    {
        if (!outer_) { c_.scoped_ = true; c_.prev_ = kChainNone; }
    }
    ~ChainScope()
    {
        if (!outer_) { c_.scoped_ = false; c_.prev_ = kChainNone; }
    }
    ChainScope(const ChainScope &) = delete;
    ChainScope &operator=(const ChainScope &) = delete;

private:
    LaunchChain &c_;
    bool outer_;
};

}  // namespace uavrl
