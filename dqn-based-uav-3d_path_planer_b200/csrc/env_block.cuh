// env_block.cuh -- the per-CTA body of the env step / observation kernel (env_kernel, env.cu): EPB envs starting at e0,
// NT threads, shared-memory scratch passed in.
// Phases and references: see env.cu.
#pragma once
#include "env.cuh"

namespace uavrl {

// The 80 probes of UAV.state_PathPlan (UAV.py:533-555,562-566) as integer offsets from the UAV position and observation
// slots: 3 grids of 5 x 5 at 1 / 5 / 10 m, then 5 points below.  Built once per CTA in shared memory (a __constant__ table
// indexed per lane would serialise); x = px + dx is the same IEEE operation probe_point performs (small integers are exact).
struct ProbeOff { signed char dx, dy, dz; unsigned char slot; };
__device__ __forceinline__ ProbeOff probe_offset(int p)
{
    ProbeOff o;
    if (p < 75) {
        const int g = p / 25, ij = p - 25 * g, i = ij / 5, j = ij - 5 * i;
        const int sc = (g == 0) ? 1 : (g == 1) ? 5 : 10;
        o.dx = (signed char)(sc * (i - 2)); o.dy = (signed char)(sc * (j - 2)); o.dz = 0; o.slot = (unsigned char)(11 + p);
    } else {
        o.dx = 0; o.dy = 0; o.dz = (signed char)(-(p - 75 + 1)); o.slot = (unsigned char)(90 + (p - 75));
    }
    return o;
}

template <int EPB>
struct EnvSmem {
    Cyl cyl[kMaxCyl];
    __align__(16) float obs[EPB][kObsDim];
    double pos[3][EPB];
    unsigned long long mask[EPB];
    uint8_t flags[EPB];                 // EXTRAS/APF: 1 = shift this env's sub-goal queue, 2 = reload it from the pool
    double st_rew[EPB];                 // statistics parked by phase 1 (reward, flags: stepped | ended<<1 | collision<<2 | success<<3 | lose<<4)
    uint8_t st_flags[EPB];
    uint8_t safe[EPB];                  // 1: none of this env's 75 planar probes can be out of bounds (phase 2 skips the test)
    ProbeOff probe[80];
};

__device__ __forceinline__ void load_scenario(const EnvDev &d, int scen, EnvRegs &s)
{
    const double *st = d.pool_start + (size_t)scen * 3;
    const double *gl = d.pool_goal + (size_t)scen * 3;
    const double *v0 = d.pool_v0 + (size_t)scen * 3;
    s.px = st[0]; s.py = st[1]; s.pz = st[2];
    s.gx = gl[0]; s.gy = gl[1]; s.gz = gl[2];
    s.vx = v0[0]; s.vy = v0[1]; s.V = v0[2];
    s.theta = angle_xy(s.vx, s.vy);
    s.score = 0.0; s.total = 0.0; s.path_len = 0.0;
    s.step = 0; s.cursor = 0; s.done = 0;
    s.n_sub = d.pool_nsub[scen];
    s.alias = d.pool_alias[scen];
}

__device__ __forceinline__ unsigned long long cull_mask(const EnvDev &d, const Cyl *cyl, double px, double py)
{
    unsigned long long m = 0ull;
    for (int c = 0; c < d.k.n_cyl; ++c) {
        const double reach = cyl[c].R + d.cull_w;
        const bool near_x = fabs(px - cyl[c].cx) <= reach;
        const bool near_y = fabs(py - cyl[c].cy) <= reach;
        if (near_x && near_y) m |= (1ull << c);
    }
    return m;
}

// The same candidate set computed by G = 32 / LPW lanes per env: lane (part, env) tests cylinders part, part + G, ... and the
// partial masks are OR-ed across the parts.  Every lane of the warp must call this (shuffles); lanes >= LPW take their env's
// position from lane (lane % LPW).
template <int LPW>
__device__ __forceinline__ unsigned long long cull_mask_coop(const EnvDev &d, const Cyl *cyl, double px, double py, int lane)
{
    constexpr int G = 32 / LPW;
    if (G == 1) return cull_mask(d, cyl, px, py);
    const unsigned full = 0xffffffffu;
    const int src = lane % LPW, part = lane / LPW;
    const double x = __shfl_sync(full, px, src), y = __shfl_sync(full, py, src);
    unsigned long long m = 0ull;
    for (int c = part; c < d.k.n_cyl; c += G) {
        const double reach = cyl[c].R + d.cull_w;
        if (fabs(x - cyl[c].cx) <= reach && fabs(y - cyl[c].cy) <= reach) m |= (1ull << c);
    }
#pragma unroll
    for (int off = LPW; off < 32; off <<= 1) m |= __shfl_xor_sync(full, m, off);
    return m;
}

__device__ __forceinline__ int threat_masked(const EnvConst &k, const Cyl *cyl, unsigned long long m,
                                             double x, double y, double z)
{
    if (out_of_bounds(k, x, y, z)) return 1;
    while (m) {
        const int c = __ffsll((long long)m) - 1;
        m &= m - 1;
        if (cyl_hit(cyl[c], x, y, z)) return 1;
    }
    return 0;
}

// USE_PDL: execute griddepcontrol.wait right before the actions are read (stand-alone kernel inside a PDL chain);
// the fused kernel has already waited.
// LPW = envs per phase-1 warp: EPB / LPW warps run the fp64 chains of LPW envs each (one lane per env).  The chain is
// latency bound, so few lanes on several warps (= several SM sub-partitions) finish sooner than 32 lanes on one warp.
// device-side UAV.cal_force over the env's obstacle table
struct ApfDev {
    static constexpr bool enabled = true;
    const ApfObs *ob; int n;
    __device__ __forceinline__ P3 force(double x, double y, double z) const { return apf_force(ob, n, x, y, z); }
};

// The episode record of env e, whose episode just ended in state s on scenario scen (uavrl_env_set_records): slot j n + e for
// its j-th finished episode, or a drop when that slot is beyond the capacity.  start2goal and planner_len are Eu_Loc_distance
// and calculate_path_len (BaseClass/CalMod.py:133-139) in the reference's order, on the pool's copy of the scenario.
__device__ __forceinline__ void write_record(const EnvDev &d, const EnvRecDev &rec, int e, int scen, const EnvRegs &s, int outcome,
                                             int steps, int coll)
{
    const int j = rec.ord[e];
    const long long slot = (long long)j * d.n + e;
    if (slot >= rec.cap) { atomicAdd(&rec.counts[1], 1ull); return; }
    const double *st = d.pool_start + (size_t)scen * 3, *gl = d.pool_goal + (size_t)scen * 3;
    const double *q = d.pool_sub + (size_t)scen * d.K * 3;
    double plen = 0.0;
    for (int i = 1; i < s.n_sub; ++i) plen = dadd(plen, dist3(q[3 * i - 3], q[3 * i - 2], q[3 * i - 1], q[3 * i], q[3 * i + 1], q[3 * i + 2]));
    uavrl_episode_record &r = rec.rec[slot];
    r.scenario = scen; r.env = e; r.ordinal = j; r.outcome = outcome;
    r.steps = steps; r.subgoals = s.cursor; r.collisions = coll; r.reserved = 0;
    r.total_score = s.total; r.path_len = s.path_len;
    r.start2goal = dist3(st[0], st[1], st[2], gl[0], gl[1], gl[2]);
    r.planner_len = plen;
    r.final_dist = dist3(s.px, s.py, s.pz, s.gx, s.gy, s.gz);
    r.energy = (d.extras & kExtraEnergy) ? d.energy[e] : 0.0;
    atomicAdd(&rec.counts[0], 1ull);
}

// EXTRAS: the optional models of uavrl_env_set_extras (energy accumulator, APF with per-env sub-goal queues, trajectory
// recording) and the episode records of uavrl_env_set_records (rec); the default instantiation (false) is the hot path and
// carries none of it.
template <bool DO_STEP, int EPB, int NT, bool USE_PDL, int LPW, bool EXTRAS = false>
__device__ __forceinline__ void env_block(const EnvDev &d, EnvSmem<EPB> &sm, int e0, int tid, int action_kind,
                                          const void *__restrict__ actions, float *__restrict__ obs, float *__restrict__ reward,
                                          uint8_t *__restrict__ done_out, uint8_t *__restrict__ info_out,
                                          uint8_t *__restrict__ coll_out, uint8_t *__restrict__ ended_out,
                                          const EnvRecDev *rec = nullptr, const EnvMotionDev *mot = nullptr,
                                          MotionSmem *msm = nullptr)
{
#define ENV_TRACE(slot) do { if (d.trace && blockIdx.x == 0 && tid == 0) d.trace[slot] = clock64(); } while (0)
    ENV_TRACE(0);
    Cyl *s_cyl = sm.cyl;
    uint8_t *sm_flags = EXTRAS ? sm.flags : nullptr;
    if (EXTRAS && tid < EPB) sm.flags[tid] = 0;
    if (tid < 80) sm.probe[tid] = probe_offset(tid);
    if (DO_STEP && tid < EPB) { sm.st_flags[tid] = 0; sm.st_rew[tid] = 0.0; }
    float (*s_obs)[kObsDim] = sm.obs;
    double (*s_pos)[EPB] = sm.pos;
    unsigned long long *s_mask = sm.mask;
    // PDL: the predecessor in the lockstep loops is the act kernel, which only writes `actions`; per-env state and
    // the pool were last written by the previous env step.  The phase-1 lanes load their state (and the sub-goals the step
    // will read) while the cylinder table is still on its way to shared memory, and wait just before they read the action;
    // the other warps have nothing to do until phase 2.
    constexpr int NW1 = EPB / LPW;
    static_assert(EPB % LPW == 0 && LPW <= 32 && NW1 * 32 <= NT, "phase-1 warp layout");
    const int wp = tid >> 5, ln = tid & 31;
    const int le = wp * LPW + ln;                            // local env of this lane (valid lanes only)
    const int e = e0 + le;
    const bool valid = (wp < NW1) && (ln < LPW) && (e < d.n);
    EnvRegs s;
    StepOut o;                                               // phase 1's outputs, written back behind the phase-1 barrier
    o.reward = 0.0; o.done_ret = 0; o.info = 0; o.coll = 0;
    uint8_t ended_flag = 0;
    // EXTRAS with records: parked = this env has no suite position left and is not stepped; park_after = its episode ended
    // and it has none for the next one, so it keeps the finished episode's state instead of an auto-reset
    bool parked = false, park_after = false;
    int scen = 0;
    P3 sgc[3];                                               // sub-goal queue entries cursor, cursor + 1, cursor + 2 (prefetched)
    s.px = 0.0; s.py = 0.0;
    if (valid) {
        s.px = d.px[e]; s.py = d.py[e]; s.pz = d.pz[e];
        s.vx = d.vx[e]; s.vy = d.vy[e]; s.V = d.V[e];
        s.score = d.score[e]; s.total = d.total[e]; s.path_len = d.path_len[e];
        s.gx = d.gx[e]; s.gy = d.gy[e]; s.gz = d.gz[e];
        s.step = d.step[e]; s.cursor = d.cursor[e]; s.n_sub = d.n_sub[e];
        s.done = d.done[e]; s.alias = d.alias[e];
        s.theta = d.theta[e];
        scen = d.scen[e];
        const bool apf_q = EXTRAS && (d.extras & kExtraApf);
        const double *q = apf_q ? d.sub_env + (size_t)e * d.K * 3 : d.pool_sub + (size_t)scen * d.K * 3;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int i = s.cursor + j;
            if (i < s.n_sub && i < d.K) { sgc[j].x = q[3 * i]; sgc[j].y = q[3 * i + 1]; sgc[j].z = q[3 * i + 2]; }
            else { sgc[j].x = 0.0; sgc[j].y = 0.0; sgc[j].z = 0.0; }
        }
        if (EXTRAS && DO_STEP && (d.extras & kExtraRecord)) parked = (long long)rec->ord[e] * d.n + e >= rec->limit;
    }
    const int cur0 = s.cursor;
    // EXTRAS with moving obstacles: every CTA stages O_t (centres into the cylinders, and the APF table at O_t with the
    // direction of each obstacle's current velocity variant); the APF reads below all take apf_tab
    const bool moving = EXTRAS && (d.extras & kExtraMotion);
    const ApfObs *apf_tab = d.apf_obs;
    if (moving) {
        for (int c = tid; c < d.k.n_cyl; c += NT) {
            const MoveObs o = mot->rd[c];
            msm->o[c] = o;
            Cyl cy = d.cyl[c];
            cy.cx = o.x; cy.cy = o.y;
            s_cyl[c] = cy;
            if (d.extras & kExtraApf) {
                ApfObs a = d.apf_obs[c];
                const int v = motion_variant(o.vx, o.vy);
                a.x = o.x; a.y = o.y; a.vx = o.vx; a.vy = o.vy;
                a.cav = mot->dir[8 * c + 2 * v]; a.sav = mot->dir[8 * c + 2 * v + 1];
                msm->apf[c] = a;
            }
        }
        apf_tab = msm->apf;
    } else {
        for (int i = tid; i < d.k.n_cyl * 6; i += NT)
            reinterpret_cast<double *>(s_cyl)[i] = reinterpret_cast<const double *>(d.cyl)[i];
    }
    __syncthreads();
    ENV_TRACE(1);
    if (USE_PDL && wp >= NW1) { pdl_wait(); pdl_trigger(); }

    if (wp < NW1) {
        unsigned long long mask = 0ull;
        double px = 0.0, py = 0.0, pz = 0.0, rew = 0.0;
        int n_stepped = 0, n_ended = 0, n_coll = 0, n_succ = 0, n_lose = 0;
        // exact candidate cull, shared by the whole warp (the lanes beyond LPW would otherwise idle)
        mask = cull_mask_coop<LPW>(d, s_cyl, s.px, s.py, ln);
        ENV_TRACE(2);
        if (valid) {
            if (DO_STEP && !(EXTRAS && parked)) {
                if (USE_PDL) { pdl_wait(); pdl_trigger(); }
                double act;
                if (action_kind == UAVRL_ACT_CONT_F32) act = (double)static_cast<const float *>(actions)[e];
                else if (action_kind == UAVRL_ACT_CONT_F64) act = static_cast<const double *>(actions)[e];
                else if (action_kind == UAVRL_ACT_CONT_F32X2) act = (double)static_cast<const float *>(actions)[2 * e];
                else act = (double)static_cast<const int32_t *>(actions)[e];
                ENV_TRACE(3);
                const int mode = (action_kind == UAVRL_ACT_DISCRETE27) ? 1 : 0;
                const bool apf_on = EXTRAS && (d.extras & kExtraApf);
                const double *q = apf_on ? d.sub_env + (size_t)e * d.K * 3 : d.pool_sub + (size_t)scen * d.K * 3;
                // entries cursor .. cursor + 2 were prefetched with the state (the step reads cursor and, after a pop, cursor + 1)
                auto sub = [q, cur0, &sgc](int i) {
                    const int j = i - cur0;
                    if (j == 0) return sgc[0];
                    if (j == 1) return sgc[1];
                    if (j == 2) return sgc[2];
                    P3 p; p.x = q[3 * i]; p.y = q[3 * i + 1]; p.z = q[3 * i + 2]; return p;
                };
                const Cyl *cyl = s_cyl;
                const EnvConst kk = d.k;
                auto threat = [&kk, cyl, mask](double x, double y, double z) {
                    return threat_masked(kk, cyl, mask, x, y, z);
                };
                if (apf_on) {
                    ApfDev apf; apf.ob = apf_tab; apf.n = d.k.n_cyl;
                    const bool alias = s.alias && s.cursor == 0;
                    step_core_apf(d.k, s, mode, act, sub, threat, apf, o);
                    if (alias && s.cursor == 0) {
                        // sub_goals[0] was the position object (RRT.py:69) and was not popped: the queue keeps the moved
                        // position (a collision rebinds position, not the entry, UAV.py:427), which phase 1b and the
                        // observation then shift.  A large APF push at the start point (a moving obstacle over it) gets here.
                        P3 m;
                        if (o.coll) {                        // the step restored the old position: move it again
                            const int kk = (int)act;
                            m.x = dadd(s.px, s.vx); m.y = dadd(s.py, s.vy);
                            m.z = mode == 1 ? dadd(s.pz, dmul((double)((kk / 3) % 3 - 1), d.k.climb)) : s.pz;
                        } else {
                            m.x = s.px; m.y = s.py; m.z = s.pz;
                        }
                        double *q0 = d.sub_env + (size_t)e * d.K * 3;
                        q0[0] = m.x; q0[1] = m.y; q0[2] = m.z;
                        sgc[0] = m;
                    }
                } else {
                    step_core(d.k, s, mode, act, sub, threat, o);
                }
                ENV_TRACE(4);
                if (EXTRAS) {
                    if (d.extras & kExtraEnergy) {
                        const double pw = fly_power(d.pw, s.V);
                        d.energy[e] = dadd(d.energy[e], pw);
                        atomicAdd(d.stat_reward + 1, pw);          // lifetime total over all UAVs (UAV.energy_cost_total summed)
                    }
                    if ((d.extras & kExtraTrack) && e < d.track_n) {           // UAV.path.append (UAV.py:432)
                        const int cur = d.path_cur[e];
                        const int np = d.path_n[cur * d.track_n + e];
                        if (np < d.track_cap) {
                            double *pp = d.path_buf + (((size_t)cur * d.track_n + e) * d.track_cap + np) * 3;
                            pp[0] = s.px; pp[1] = s.py; pp[2] = s.pz;
                        }
                        d.path_n[cur * d.track_n + e] = np + 1;
                        if (s.done) { d.path_cur[e] = cur ^ 1; d.path_n[(cur ^ 1) * d.track_n + e] = 0; }     // UAV.reset: path = []
                    }
                    if (d.extras & kExtraRecord) {                  // the episode's record, before the auto-reset below
                        const int steps = rec->steps[e] + 1, coll = rec->coll[e] + o.coll;
                        if (s.done) {
                            write_record(d, *rec, e, scen, s, o.info, steps, coll);
                            const int j = rec->ord[e] + 1;
                            rec->ord[e] = j; rec->steps[e] = 0; rec->coll[e] = 0;
                            park_after = (long long)j * d.n + e >= rec->limit;
                        } else {
                            rec->steps[e] = steps; rec->coll[e] = coll;
                        }
                    }
                    if (sm_flags) sm_flags[le] = (uint8_t)((d.auto_reset && s.done && !(EXTRAS && park_after)) ? 2 : 1);   // 2: reload the queue, 1: shift it
                }
                rew = o.reward;
                n_stepped = 1; n_coll = o.coll; n_ended = s.done;
                n_succ = (o.info == 1); n_lose = (o.info == 2);
                ended_flag = (uint8_t)s.done;
                if (d.auto_reset && s.done && !(EXTRAS && park_after)) {       // UAV.reset() at the episode boundary
                    scen = (int)(((long long)scen + d.reset_stride) % d.P);
                    if (EXTRAS && (d.extras & kExtraEnergy)) d.energy[e] = 0.0;
                    load_scenario(d, scen, s);
                    mask = cull_mask(d, s_cyl, s.px, s.py);
                    d.scen[e] = scen;
                    d.gx[e] = s.gx; d.gy[e] = s.gy; d.gz[e] = s.gz;
                    d.n_sub[e] = s.n_sub;
                }
            }
            ENV_TRACE(5);
            if (obs) {
                const bool apf_on = EXTRAS && (d.extras & kExtraApf);
                // APF: an env that did not restart reads its own queue, whose entries phase 1b shifts right after this
                // (same function, so the on-the-fly shift below equals what will be stored); a restarted env reads the pool
                const bool own_q = apf_on && !(DO_STEP && d.auto_reset && n_ended && !(EXTRAS && park_after));
                const double *q = own_q ? d.sub_env + (size_t)e * d.K * 3 : d.pool_sub + (size_t)scen * d.K * 3;
                const bool shift = own_q && DO_STEP;
                const ApfObs *aob = apf_tab; const int an = d.k.n_cyl;
                const bool same_q = !(DO_STEP && d.auto_reset && n_ended && !(EXTRAS && park_after));   // still the queue the prefetch read
                auto sub = [q, shift, aob, an, same_q, cur0, &sgc](int i) {
                    P3 p;
                    const int j = i - cur0;
                    if (same_q && j >= 0 && j <= 2) p = (j == 0) ? sgc[0] : (j == 1) ? sgc[1] : sgc[2];
                    else { p.x = q[3 * i]; p.y = q[3 * i + 1]; p.z = q[3 * i + 2]; }
                    if (EXTRAS && shift) { const P3 f = apf_force(aob, an, p.x, p.y, p.z); p.x = dadd(p.x, f.x); p.y = dadd(p.y, f.y); p.z = dadd(p.z, f.z); }
                    return p;
                };
                obs_scalars(s, sub, &s_obs[le][0]);
            }
            ENV_TRACE(6);
            px = s.px; py = s.py; pz = s.pz;
        }
        if (ln < LPW) {
            s_pos[0][le] = px; s_pos[1][le] = py; s_pos[2][le] = pz;
            s_mask[le] = mask;
            // Bounds shortcut for the 75 planar probes (offsets within +-20 m, z = pz): IEEE addition is monotonic in the
            // offset, so if px-20 and px+20 (as rounded sums) are inside [0, width] every px+dx is, likewise y; z is pz
            // itself.  Then PathPlan_City.py:218 is false for all of them and phase 2 need not evaluate it.
            sm.safe[le] = (uint8_t)(!(dadd(px, -20.0) < 0.0) && !(dadd(px, 20.0) > d.k.width) && !(dadd(py, -20.0) < 0.0) &&
                                    !(dadd(py, 20.0) > d.k.width) && !(pz < 0.0) && !(pz > d.k.h));
        }
        // running statistics: parked per env, reduced by the last warp after the observation tile is out (off the chain)
        if (DO_STEP && valid) {
            sm.st_rew[le] = rew;
            sm.st_flags[le] = (uint8_t)(n_stepped | (n_ended << 1) | (n_coll << 2) | (n_succ << 3) | (n_lose << 4));
        }
    }
    ENV_TRACE(7);
    __syncthreads();
    ENV_TRACE(8);
    // write-back of the stepped state and the step's outputs: behind the barrier, i.e. while the other warps already probe
    // (these ~25 stores per env used to sit between the step and the barrier every warp of the CTA waits at)
    if (DO_STEP && valid && !(EXTRAS && parked)) {
        if (reward) reward[e] = (float)o.reward;
        d.rew64[e] = o.reward;
        if (done_out) done_out[e] = (uint8_t)o.done_ret;
        if (info_out) info_out[e] = (uint8_t)o.info;
        if (coll_out) coll_out[e] = (uint8_t)o.coll;
        if (ended_out) ended_out[e] = ended_flag;
        d.px[e] = s.px; d.py[e] = s.py; d.pz[e] = s.pz;
        d.vx[e] = s.vx; d.vy[e] = s.vy; d.V[e] = s.V; d.theta[e] = s.theta;
        d.score[e] = s.score; d.total[e] = s.total; d.path_len[e] = s.path_len;
        d.step[e] = s.step; d.cursor[e] = s.cursor;
        d.done[e] = (uint8_t)s.done; d.alias[e] = (uint8_t)s.alias;
    }
    if (moving && DO_STEP) {
        // every obstacle runs once: O_{t+1}, the same arithmetic in every CTA, for the probes of phase 2; CTA 0 stores it into
        // the buffer the next step reads (this launch reads the other one).  msm->apf keeps O_t for phase 1b.
        for (int c = tid; c < d.k.n_cyl; c += NT) {
            MoveObs o = msm->o[c];
            obstacle_run(o, mot->len, mot->width);
            s_cyl[c].cx = o.x; s_cyl[c].cy = o.y;
            if (blockIdx.x == 0) mot->wr[c] = o;
        }
        __syncthreads();
    }
    if (EXTRAS && DO_STEP && (d.extras & kExtraApf)) {
        // phase 1b, all threads: UAV.Adjust_subgoal (UAV.py:156-166) for the stored queues -- every entry moves by the
        // force at its (pre-step) position; an env that restarted takes its new scenario's queue instead
        for (int idx = tid; idx < EPB * d.K; idx += NT) {
            const int le = idx / d.K, i = idx - le * d.K, e = e0 + le;
            if (e >= d.n || sm.flags[le] == 0) continue;
            double *q = d.sub_env + ((size_t)e * d.K + i) * 3;
            if (sm.flags[le] == 2) {
                const double *src = d.pool_sub + ((size_t)d.scen[e] * d.K + i) * 3;
                q[0] = src[0]; q[1] = src[1]; q[2] = src[2];
            } else if (i < d.n_sub[e]) {
                const P3 f = apf_force(apf_tab, d.k.n_cyl, q[0], q[1], q[2]);
                q[0] = dadd(q[0], f.x); q[1] = dadd(q[1], f.y); q[2] = dadd(q[2], f.z);
            }
        }
    }
    auto flush_stats = [&]() {
        if (!DO_STEP || wp != NT / 32 - 1) return;
        const unsigned full = 0xffffffffu;
        const int fl = (ln < EPB) ? (int)sm.st_flags[ln] : 0;
        double rew = (ln < EPB) ? sm.st_rew[ln] : 0.0;
        int n_stepped = fl & 1, n_ended = (fl >> 1) & 1, n_coll = (fl >> 2) & 1, n_succ = (fl >> 3) & 1, n_lose = (fl >> 4) & 1;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            n_stepped += __shfl_xor_sync(full, n_stepped, off);
            n_ended += __shfl_xor_sync(full, n_ended, off);
            n_coll += __shfl_xor_sync(full, n_coll, off);
            n_succ += __shfl_xor_sync(full, n_succ, off);
            n_lose += __shfl_xor_sync(full, n_lose, off);
            rew += __shfl_xor_sync(full, rew, off);
        }
        if (ln == 0 && n_stepped) {
            atomicAdd(&d.stat_counts[0], (unsigned long long)n_stepped);
            if (n_ended) atomicAdd(&d.stat_counts[1], (unsigned long long)n_ended);
            if (n_coll) atomicAdd(&d.stat_counts[2], (unsigned long long)n_coll);
            if (n_succ) atomicAdd(&d.stat_counts[3], (unsigned long long)n_succ);
            if (n_lose) atomicAdd(&d.stat_counts[4], (unsigned long long)n_lose);
            atomicAdd(d.stat_reward, rew);
        }
    };
    if (!obs) { flush_stats(); return; }

    // phase 2: occupancy probes
    for (int idx = tid; idx < EPB * 80; idx += NT) {
        const int le = idx / 80, p = idx - 80 * le;
        if (e0 + le >= d.n) break;
        const ProbeOff po = sm.probe[p];
        const double x = dadd(s_pos[0][le], (double)po.dx), y = dadd(s_pos[1][le], (double)po.dy);
        const double z = (p < 75) ? s_pos[2][le] : dadd(s_pos[2][le], (double)po.dz);
        int hit = (p < 75 && sm.safe[le]) ? 0 : out_of_bounds(d.k, x, y, z);
        unsigned long long m = s_mask[le];
        while (m && !hit) {
            const int c = __ffsll((long long)m) - 1;
            m &= m - 1;
            hit = cyl_hit(s_cyl[c], x, y, z);
        }
        s_obs[le][po.slot] = hit ? 1.0f : 0.0f;
    }
    ENV_TRACE(9);
    __syncthreads();
    ENV_TRACE(10);

    // phase 3: coalesced 16-byte stores of the contiguous [nvalid][100] tile
    const int nvalid = min(EPB, d.n - e0);
    const int nvec = nvalid * (kObsDim / 4);
    float4 *dst = reinterpret_cast<float4 *>(obs + (size_t)e0 * kObsDim);
    const float4 *src = reinterpret_cast<const float4 *>(&s_obs[0][0]);
    for (int i = tid; i < nvec; i += NT) dst[i] = src[i];
    flush_stats();
    ENV_TRACE(11);
}

}  // namespace uavrl
