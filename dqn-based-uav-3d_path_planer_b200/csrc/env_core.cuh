// env_core.cuh -- per-UAV step / observation arithmetic of the PathPlan_City hot path.
//
// One instance of this code runs per env inside env_step_kernel (env.cu).  It is written as
// host/device inline functions so the *same source* can also be compiled for the host by the
// CPU-side logic test (tests/host_shim) and by the host scenario generator's collision test;
// the product's step path is the CUDA kernel only.
//
// Arithmetic contract (DESIGN.md "numerics"): state and reward in fp64 like the Python reference;
// every +,-,*,/,sqrt that feeds an integer predicate (collision, bounds, termination) is an
// explicitly rounded IEEE op (no FMA contraction) in the reference's operation order, so given
// identical inputs the masks are bit-identical to the reference's.  Transcendentals
// (atan2/sin/cos) come from the CUDA math library (<= 2 ulp from glibc's): positions agree to
// ~1e-15 relative, far inside the 1e-5 tolerance.
//
// Reference: Agents/UAV.py:397-567, Envs/PathPlan_City.py:215-223, Obstacles/building.py:20-26,
// BaseClass/CalMod.py:64-65,89-102.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define UAVRL_HD __host__ __device__ __forceinline__
#else
#define UAVRL_HD inline
#endif

namespace uavrl {

#if defined(__CUDA_ARCH__)
UAVRL_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
UAVRL_HD double dsub(double a, double b) { return __dsub_rn(a, b); }
UAVRL_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
UAVRL_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
UAVRL_HD double dsqrt(double a) { return __dsqrt_rn(a); }
#else
// host build: compiled with -ffp-contract=off
UAVRL_HD double dadd(double a, double b) { return a + b; }
UAVRL_HD double dsub(double a, double b) { return a - b; }
UAVRL_HD double dmul(double a, double b) { return a * b; }
UAVRL_HD double ddiv(double a, double b) { return a / b; }
UAVRL_HD double dsqrt(double a) { return sqrt(a); }
#endif

constexpr double kPi = 3.14159265358979323846;
constexpr int kObsDim = 100;

struct Cyl {            // building.py:8-11 plus a guard band around R^2 for the sqrt-free fast path
    double cx, cy, R, H, r2lo, r2hi;
};

struct EnvConst {
    double width, h;                    // PathPlan_City.py:218 tests x AND y against `width`
    double max_v, min_v, steering, climb;
    int32_t max_step;
    int32_t n_cyl;
};

struct EnvRegs {
    double px, py, pz, vx, vy, V, score, total, path_len, gx, gy, gz;
    double theta;                       // calculate_angle(0, V_vector) of the current V_vector
    int32_t step, cursor, n_sub;
    int32_t done, alias;
};

struct StepOut {
    double reward;
    int32_t done_ret, info, coll;
};

struct P3 { double x, y, z; };

// CalMod.py:64-65  sqrt((dx)**2 + (dy)**2 + (dz)**2), left-to-right
UAVRL_HD double dist3(double ax, double ay, double az, double bx, double by, double bz)
{
    const double dx = dsub(ax, bx), dy = dsub(ay, by), dz = dsub(az, bz);
    return dsqrt(dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz)));
}

// CalMod.py:89-102 (mod=1): atan2 -> degrees -> (a + 360) % 360 / 180 * pi.
// a+360 lies in [180,540], where Python's float % 360 is exactly "subtract 360 if >= 360".
UAVRL_HD double angle_xy(double dx, double dy)
{
    double a = atan2(dy, dx);
    a = dmul(a, 180.0 / kPi);
    double t = dadd(a, 360.0);
    t = (t >= 360.0) ? dsub(t, 360.0) : t;
    return dmul(ddiv(t, 180.0), kPi);
}

// cos|calculate_angle(a) - calculate_angle(b)| for two planar vectors WITHOUT the angles: the reference forms both angles with
// atan2 -> degrees -> (+360) % 360 -> radians and takes the cosine of their difference (UAV.py:422-423,435,488-490), which
// is the cosine of the angle between the vectors = their normalised dot product (the % 360 wrap and |.| do not change a
// cosine).  calculate_angle of a zero vector is atan2 of its signed zeros: atan2(+-0, -0) = +-pi, the direction (-1, 0),
// and atan2(+-0, +0) = +-0, the direction (1, 0).  A zero V_vector carries the signs of speed 0 times (cos, sin), so both
// occur.  Agrees with the literal evaluation to a few 1e-16 (both are ~1 ulp evaluations of the same real number); nothing
// but the reward depends on it.
// UAVRL_LITERAL_ANGLES=1 compiles the literal atan2 / cos chain instead (about 400 more dependent fp64 instructions per step).
#ifndef UAVRL_LITERAL_ANGLES
#define UAVRL_LITERAL_ANGLES 0
#endif
UAVRL_HD double cos_between(double ax, double ay, double bx, double by)
{
    double na = dsqrt(dadd(dmul(ax, ax), dmul(ay, ay)));
    double nb = dsqrt(dadd(dmul(bx, bx), dmul(by, by)));
    if (na == 0.0) { ax = copysign(1.0, ax); ay = 0.0; na = 1.0; }
    if (nb == 0.0) { bx = copysign(1.0, bx); by = 0.0; nb = 1.0; }
    return ddiv(dadd(dmul(ax, bx), dmul(ay, by)), dmul(na, nb));
}

// calculate_angle(0, V_vector) of V_vector = V * (cos t, sin t), V > 0: t wrapped into [0, 2 pi) -- what the reference's
// atan2 -> degrees -> % 360 -> radians round trip returns up to its own rounding (~1e-15).  One wrap covers |t| < 4 pi minus
// the old heading, i.e. |a0 * steering| < 2 pi; beyond that the step takes the angle of V_vector itself (heading_of).
UAVRL_HD double wrap_2pi(double t)
{
    if (t < 0.0) t = dadd(t, 2.0 * kPi);
    if (t >= 2.0 * kPi) t = dsub(t, 2.0 * kPi);
    return t;
}

// The cached heading after a step that set V_vector = speed * (cos t, sin t) (speed >= 0, uavrl_env_create refuses a
// negative Min_V): t wrapped once when that lands in [0, 2 pi), else calculate_angle(0, V_vector) itself -- a zero
// V_vector (speed 0) or a turn of 2 pi or more, which one wrap cannot bring back.
UAVRL_HD double heading_of(double t, double V, double vx, double vy)
{
    const double w = wrap_2pi(t);
    return (V > 0.0 && w >= 0.0 && w < 2.0 * kPi) ? w : angle_xy(vx, vy);
}

// The reference evaluates calculate_angle(0, V_vector) three times per step on the SAME vector
// (seta_old at :411 is last step's value, tri_V at :423 and state[7] at :526 are this step's):
// EnvRegs.theta caches it -- identical value, one atan2 instead of three.

// building.py:20-26 -- strict `z > H` and strict `dist < R`
UAVRL_HD int cyl_hit(const Cyl &c, double x, double y, double z)
{
    if (z > c.H) return 0;
    const double dx = dsub(x, c.cx), dy = dsub(y, c.cy);
    const double s = dadd(dmul(dx, dx), dmul(dy, dy));      // (+ 0.0**2 for the z term: exact no-op)
    if (s < c.r2lo) return 1;
    if (s > c.r2hi) return 0;
    return dsqrt(s) < c.R;                                   // the reference's exact predicate
}

// PathPlan_City.py:218 (inclusive upper bounds, y against width)
UAVRL_HD int out_of_bounds(const EnvConst &k, double x, double y, double z)
{
    return (x < 0.0) | (x > k.width) | (y < 0.0) | (y > k.width) | (z < 0.0) | (z > k.h);
}

// UAV.py:246-253 Calc_V
UAVRL_HD double calc_v(const EnvConst &k, double &vx, double &vy)
{
    double V = dsqrt(dadd(dadd(dmul(vx, vx), dmul(vy, vy)), 0.0));
    if (V > k.max_v) {
        const double f = ddiv(k.max_v, V);
        vx = dmul(vx, f);
        vy = dmul(vy, f);
        V = k.max_v;
    }
    return V;
}

// UAV.py:239-245 Calc_Fly_Power with the constants of config/UAV.xml <Power_param><Fly_power> (SURVEY 8a-8).
struct PowerConst { double P_i, v_0, d_0, rho, s, A, P_b, F_b, xi; };
UAVRL_HD double fly_power(const PowerConst &c, double V)
{
    const double V2 = dmul(V, V), v02 = dmul(c.v_0, c.v_0);
    const double V4 = dmul(V2, V2), v04 = dmul(v02, v02);
    const double induced = dmul(c.P_i, dsqrt(dsub(dsqrt(dadd(1.0, ddiv(V4, dmul(4.0, v04)))), ddiv(V2, dmul(2.0, v02)))));
    const double parasite = dmul(dmul(dmul(dmul(dmul(0.5, c.d_0), c.rho), c.s), c.A), dmul(V2, V));
    const double blade = dmul(dmul(c.xi, c.P_b), dadd(1.0, ddiv(dmul(3.0, V2), dmul(c.F_b, c.F_b))));
    return dadd(dadd(induced, parasite), blade);
}

// Moving obstacle as the APF code sees it (UAV.py:174-210): position, radius, velocity `v`, and -- constant per obstacle --
// |v| and cos/sin of calculate_angle(0, v), evaluated once on the host.
struct ApfObs { double x, y, z, R, vx, vy, vz, vmag, cav, sav; };

// UAV.cal_force (UAV.py:174-210): repulsion min(1, R/d_edge^2) (max(-d_edge, 2) inside the obstacle) along -(p -> centre)
// plus the motion force min(1, |v| R / d_edge^2) along v, for obstacles with v != 0 whose edge is within 60 m.
// When the accumulated magnitude exceeds 100 the reference calls Cal_SubTask_Dynamic() without its two arguments (a
// TypeError): here the force accumulated so far is returned (documented deviation; needs > 50 obstacles in range).
UAVRL_HD P3 apf_force(const ApfObs *ob, int n, double px, double py, double pz)
{
    P3 tot; tot.x = 0.0; tot.y = 0.0; tot.z = 0.0;
    double cum = 0.0;
    for (int i = 0; i < n; ++i) {
        const ApfObs &o = ob[i];
        if (o.vx == 0.0 && o.vy == 0.0 && o.vz == 0.0) continue;            // :180-182
        const double dis = dist3(px, py, pz, o.x, o.y, o.z);                  // :183
        const double d2e = dsub(dis, o.R);                                    // :185
        if (d2e > 60.0) continue;                                             // :186-187
        const double dd = dmul(d2e, d2e);
        double f1 = ddiv(o.R, dd);                                            // :190  min(1, w R / d^2), w = 1
        f1 = (1.0 < f1 || f1 != f1) ? 1.0 : f1;
        const double a1 = angle_xy(dsub(o.x, px), dsub(o.y, py));             // :191
        if (d2e < 0.0) f1 = (-d2e > 2.0) ? -d2e : 2.0;                        // :196-197
        const double f1x = dmul(-f1, cos(a1)), f1y = dmul(-f1, sin(a1));      // :198
        double f2 = ddiv(dmul(o.vmag, o.R), dd);                              // :200
        f2 = (1.0 < f2 || f2 != f2) ? 1.0 : f2;
        const double f2x = dmul(f2, o.cav), f2y = dmul(f2, o.sav);            // :201
        cum = dadd(cum, dadd(f1, f2));                                        // :202
        tot.x = dadd(dadd(tot.x, f1x), f2x);                                  // :203
        tot.y = dadd(dadd(tot.y, f1y), f2y);
        if (cum > 100.0) return tot;                                          // :205-208 (see above)
    }
    return tot;
}

// Moving obstacles (uavrl_env_set_motion): a cylinder's centre and planar velocity.  z, R and H are fixed.
struct MoveObs { double x, y, vx, vy; };

// One obstacle's run() (the reference's per-obstacle hook, Obstacles/BaseThreaten.py, is `pass`; this is the port's rule):
// x' = x + vx, reflected once at 0 and at len (y likewise at width), and the velocity component reverses at a reflection.
// One reflection suffices because centres lie in [0, len] x [0, width] with |vx| <= len, |vy| <= width.
UAVRL_HD void obstacle_run(MoveObs &o, double len, double width)
{
    double x = dadd(o.x, o.vx);
    if (x < 0.0) { x = -x; o.vx = -o.vx; }
    else if (x > len) { x = dsub(len, dsub(x, len)); o.vx = -o.vx; }
    double y = dadd(o.y, o.vy);
    if (y < 0.0) { y = -y; o.vy = -o.vy; }
    else if (y > width) { y = dsub(width, dsub(y, width)); o.vy = -o.vy; }
    o.x = x; o.y = y;
}

// Which of an obstacle's four sign variants (+-vx, +-vy) its velocity is in: a reflection only flips a sign bit, so the APF
// direction of every variant is evaluated once on the host and the step selects it by the current signs.
UAVRL_HD int motion_variant(double vx, double vy) { return (signbit(vx) ? 1 : 0) | (signbit(vy) ? 2 : 0); }

struct NoApf {
    static constexpr bool enabled = false;
    UAVRL_HD P3 force(double, double, double) const { P3 z; z.x = z.y = z.z = 0.0; return z; }
};

// UAV.py:397-513 update_PathPlan.  sub(i) returns entry i of this env's sub-goal queue;
// threat(x,y,z) is PathPlan_City.Threaten_rate.  act_mode: 0 continuous (action = a0), 1 discrete-27.
// apf: NoApf, or a functor with enabled = true and force(x, y, z) = UAV.cal_force at that point (APF_Enabled, UAV.py:448-453).
template <class SubFn, class ThreatFn, class ApfFn>
UAVRL_HD void step_core_apf(const EnvConst &k, EnvRegs &s, int act_mode, double action, SubFn sub,
                            ThreatFn threat, const ApfFn &apf, StepOut &o)
{
    double r = 0.0;
    o.coll = 0;
    if (s.n_sub - s.cursor == 0) {                                   // :400-406
        s.done = 1;
        r = dadd(r, (double)(k.max_step - s.step));
        s.score = dadd(s.score, r);
        o.reward = r; o.done_ret = 1; o.info = 1;
        return;
    }
    double a0 = action, dz = 0.0, speed = k.max_v;
    if (act_mode == 1) {
        const int kk = (int)action;
        const int i = kk / 9, j = (kk / 3) % 3, l = kk % 3;
        a0 = (double)(i - 1);
        dz = dmul((double)(j - 1), k.climb);
        speed = (l == 0) ? k.min_v : (l == 1) ? ddiv(dadd(k.min_v, k.max_v), 2.0) : k.max_v;
    }
    const bool alias = s.alias && s.cursor == 0;                     // sub_goals[0] IS position (RRT.py:69)
    P3 sg = sub(s.cursor);
    if (alias) { sg.x = s.px; sg.y = s.py; sg.z = s.pz; }

    s.step += 1;                                                     // :408
    const double ox = s.px, oy = s.py, oz = s.pz;                    // :409
    const double seta_old = s.theta;                                 // :411 (cached angle_xy(vx, vy))
    const double dis_old = dist3(s.px, s.py, s.pz, sg.x, sg.y, sg.z);        // :412
    const double dg_old = dist3(s.px, s.py, s.pz, s.gx, s.gy, s.gz);         // :413
    const double seta_new = dadd(seta_old, dmul(a0, k.steering));    // :414
    double sn, cs;
#if defined(__CUDA_ARCH__)
    sincos(seta_new, &sn, &cs);
#else
    sn = sin(seta_new); cs = cos(seta_new);
#endif
    s.vx = dmul(speed, cs);                                          // :415
    s.vy = dmul(speed, sn);                                          // :416
    s.V = calc_v(k, s.vx, s.vy);                                     // :417
    s.px = dadd(s.px, s.vx);                                         // :419
    s.py = dadd(s.py, s.vy);                                         // :420
    if (act_mode == 1) s.pz = dadd(s.pz, dz);
    if (alias) { sg.x = s.px; sg.y = s.py; sg.z = s.pz; }            // the aliased sub-goal moved too
#if UAVRL_LITERAL_ANGLES
    const double tri_goal = angle_xy(dsub(sg.x, s.px), dsub(sg.y, s.py));    // :422
    s.theta = angle_xy(s.vx, s.vy);
    double tri_V = s.theta;                                          // :423
#else
    const double tgx = dsub(sg.x, s.px), tgy = dsub(sg.y, s.py);     // :422 tri_goal = the direction of this vector
    s.theta = heading_of(seta_new, s.V, s.vx, s.vy);
    double tvx = s.vx, tvy = s.vy;                                   // :423 tri_V = the direction of V_vector
#endif
    if (threat(s.px, s.py, s.pz)) {                                  // :425
        r = dsub(r, 0.3);
        s.px = ox; s.py = oy; s.pz = oz;                             // :427
#if UAVRL_LITERAL_ANGLES
        tri_V = angle_xy(dsub(sg.x, s.px), dsub(sg.y, s.py));        // :428
#else
        tvx = dsub(sg.x, s.px); tvy = dsub(sg.y, s.py);              // :428
#endif
        o.coll = 1;
    }
    const double dis_new = dist3(s.px, s.py, s.pz, sg.x, sg.y, sg.z);        // :429
    const double dg_new = dist3(s.px, s.py, s.pz, s.gx, s.gy, s.gz);         // :430
    r = dsub(r, dmul(0.13, fabs(a0)));                               // :434
#if UAVRL_LITERAL_ANGLES
    r = dadd(r, dmul(0.2, cos(fabs(dsub(tri_goal, tri_V)))));        // :435
#else
    r = dadd(r, dmul(0.2, cos_between(tgx, tgy, tvx, tvy)));         // :435
#endif
    r = dadd(r, dmul(0.4, dsub(dis_old, dis_new)));                  // :436
    r = dadd(r, dmul(0.4, dsub(dg_old, dg_new)));                    // :437
    r = dsub(r, 0.1);                                                // :438
    r = dsub(r, dmul(0.01, fabs(dsub(s.pz, sg.z))));                 // :440
    s.path_len = dadd(s.path_len, s.V);                              // :443
    // :448-453 APF.  With static obstacles (the shipped config) every force is exactly 0 (UAV.py:180-182) and this block is
    // compiled out (NoApf).  Otherwise: Adjust_subgoal shifts every remaining sub-goal by the force at its position (the
    // caller applies the same shift to the stored queue), then the force at the UAV adds 0.2 |F| cos|angle(F) - tri_V|.
    double dis_t = dis_new;                                          // |p - sub_goals[0]| as the termination tests see it
    if (ApfFn::enabled) {
        const P3 f0 = apf.force(sg.x, sg.y, sg.z);                   // :449 (the aliased entry becomes a new Loc here)
        sg.x = dadd(sg.x, f0.x); sg.y = dadd(sg.y, f0.y); sg.z = dadd(sg.z, f0.z);
        const P3 F = apf.force(s.px, s.py, s.pz);                    // :450
        const double force = dist3(0.0, 0.0, 0.0, F.x, F.y, F.z);    // :451
#if UAVRL_LITERAL_ANGLES
        const double tri_force = angle_xy(F.x, F.y);                 // :452
        r = dadd(r, dmul(dmul(0.2, force), cos(fabs(dsub(tri_force, tri_V)))));     // :453
#else
        r = dadd(r, dmul(dmul(0.2, force), cos_between(F.x, F.y, tvx, tvy)));       // :452-453
#endif
        dis_t = dist3(s.px, s.py, s.pz, sg.x, sg.y, sg.z);
    }

    if (s.step >= k.max_step) {                                      // :456-465
        s.done = 1;
        r = dadd(r, dsub(50.0, dis_t));
        s.score = dadd(s.score, r); s.total = dadd(s.total, r);
        o.reward = r; o.done_ret = 1; o.info = 2;
    } else if (dis_t < 7.0 || dg_new < dist3(sg.x, sg.y, sg.z, s.gx, s.gy, s.gz)) {   // :466
        r = dadd(r, dsub(50.0, dis_t));                              // :468
        s.cursor += 1;                                               // :469
        if (s.n_sub - s.cursor == 0) {                               // :470-483
            r = dadd(r, 50.0);
            s.done = 1;
            r = dadd(r, (double)(k.max_step - s.step));
            s.score = dadd(s.score, r); s.total = dadd(s.total, r);
            o.reward = r; o.done_ret = 1; o.info = 1;
        } else {                                                     // :484-495
            s.step = 0; s.score = 0.0;                               // local reset :329-332
            s.V = calc_v(k, s.vx, s.vy);
            P3 ng = sub(s.cursor);
            if (ApfFn::enabled) {                                    // the stored queue is shifted after this call returns
                const P3 fn = apf.force(ng.x, ng.y, ng.z);
                ng.x = dadd(ng.x, fn.x); ng.y = dadd(ng.y, fn.y); ng.z = dadd(ng.z, fn.z);
            }
#if UAVRL_LITERAL_ANGLES
            const double tg = angle_xy(dsub(ng.x, s.px), dsub(ng.y, s.py));   // :488
            const double tv = s.theta;                               // :489 (V_vector unchanged by the local reset)
            r = dadd(r, dmul(0.2, cos(fabs(dsub(tg, tv)))));         // :490
#else
            r = dadd(r, dmul(0.2, cos_between(dsub(ng.x, s.px), dsub(ng.y, s.py), s.vx, s.vy)));   // :488-490
#endif
            r = dadd(r, (double)(k.max_step - s.step));              // :491
            s.score = dadd(s.score, r); s.total = dadd(s.total, r);
            o.reward = r; o.done_ret = 1; o.info = 1;
        }
    } else if (dg_new < 7.0) {                                       // :496-509
        s.done = 1;
        r = dadd(r, 50.0);
        r = dadd(r, (double)(k.max_step - s.step));
        s.score = dadd(s.score, r); s.total = dadd(s.total, r);
        o.reward = r; o.done_ret = 1; o.info = 1;
    } else {                                                         // :510-513
        s.score = dadd(s.score, r); s.total = dadd(s.total, r);
        o.reward = r; o.done_ret = 0; o.info = 0;
    }
    s.alias = 0;
}

template <class SubFn, class ThreatFn>
UAVRL_HD void step_core(const EnvConst &k, EnvRegs &s, int act_mode, double action, SubFn sub,
                        ThreatFn threat, StepOut &o)
{
    step_core_apf(k, s, act_mode, action, sub, threat, NoApf(), o);
}

// UAV.py:515-531,557-560: the 20 real-valued entries of the observation (probes are separate).
// `o` points at this env's 100 floats (stride 1).
// Outputs only (rounded to fp32 afterwards): x/10 is computed as x*0.1, within 1 fp64 ulp of the division.
UAVRL_HD double tenth(double x) { return dmul(x, 0.1); }

template <class SubFn>
UAVRL_HD void obs_scalars(const EnvRegs &s, SubFn sub, float *o)
{
    const int nleft = s.n_sub - s.cursor;
    o[0] = (float)dmul((double)s.step, 0.01);                       // :518
    float o1 = 0.f, o2 = 0.f, o3 = 0.f, o8 = 0.f, o9 = 0.f, o10 = 0.f;
    if (nleft >= 1) {                                                // :519-522
        P3 sg = sub(s.cursor);
        if (s.alias && s.cursor == 0) { sg.x = s.px; sg.y = s.py; sg.z = s.pz; }
        o1 = (float)tenth(dsub(sg.x, s.px));
        o2 = (float)tenth(dsub(sg.y, s.py));
        o3 = (float)tenth(dsub(sg.z, s.pz));
    }
    if (nleft >= 2) {                                                // :528-531
        const P3 s1 = sub(s.cursor + 1);
        o8 = (float)tenth(dsub(s1.x, s.px));
        o9 = (float)tenth(dsub(s1.y, s.py));
        o10 = (float)tenth(dsub(s1.z, s.pz));
    }
    o[1] = o1; o[2] = o2; o[3] = o3;
    o[4] = (float)s.V;                                               // :523
    o[5] = (float)s.vx; o[6] = (float)s.vy;
    o[7] = (float)s.theta;                                           // :526
    o[8] = o8; o[9] = o9; o[10] = o10;
    o[86] = (float)tenth(dsub(s.gx, s.px));                     // :557-559
    o[87] = (float)tenth(dsub(s.gy, s.py));
    o[88] = (float)tenth(dsub(s.gz, s.pz));
    o[89] = (float)tenth(s.pz);                                 // :560
    o[95] = 0.f; o[96] = 0.f; o[97] = 0.f; o[98] = 0.f; o[99] = 0.f;
}

// probe p in 0..79 -> test point and observation slot (UAV.py:533-555,562-566)
UAVRL_HD void probe_point(int p, double px, double py, double pz, double &x, double &y, double &z, int &slot)
{
    if (p < 75) {
        const int g = p / 25, ij = p - 25 * g, i = ij / 5, j = ij - 5 * i;
        const int sc = (g == 0) ? 1 : (g == 1) ? 5 : 10;
        x = dadd(px, (double)(sc * (i - 2)));
        y = dadd(py, (double)(sc * (j - 2)));
        z = pz;
        slot = 11 + p;
    } else {
        const int kdn = p - 75;
        x = px; y = py;
        z = dsub(pz, (double)(kdn + 1));
        slot = 90 + kdn;
    }
}

}  // namespace uavrl
