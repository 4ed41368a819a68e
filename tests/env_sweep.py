"""Shared pieces of the env sweeps (test_env_shapes_gpu.py, test_motion_shapes_gpu.py): generated cities, hand-made scenario
pools, the seek policy, the oracle's auto-reset, the observation comparison with the heading on the circle, the energy
model's constants and UAV parameter sets."""
import numpy as np
import torch

import oracle as O
from gpu_util import assert_obs

F64 = ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len")


# ----------------------------------------------------------------------------------------------------------- cities
def make_city(kind, seed=0):
    """(length, width, h, buildings [n, 5] = cx, cy, base z, R, H) of a generated city."""
    rng = np.random.default_rng(seed)
    if kind == "empty":                                   # only the bounds; the kernel allocates one dummy cylinder
        return 500.0, 500.0, 100.0, np.zeros((0, 5))
    if kind == "one":
        return 500.0, 500.0, 100.0, np.array([[250.0, 250.0, 0.0, 40.0, 60.0]])
    if kind == "dense64":
        # 64 overlapping cylinders around the centre (one probe sees several candidates, bit 63 is set), a few straddling the
        # box edge, some taller than h, some lower than the probe heights, non-zero base z
        b = np.zeros((64, 5))
        b[:, 0] = rng.uniform(150, 350, 64); b[:, 1] = rng.uniform(150, 350, 64)
        b[:, 2] = rng.uniform(0.0, 4.0, 64); b[:, 3] = rng.uniform(6, 22, 64); b[:, 4] = rng.uniform(5, 140, 64)
        b[:4, :2] = [[-6, 100], [505, 300], [200, -3], [300, 502]]
        b[60:, 4] = rng.uniform(0.5, 4.0, 4)              # below most probe heights
        b[63] = (250.0, 250.0, 1.0, 25.0, 120.0)          # bit 63, in the middle of the pack
        return 500.0, 500.0, 100.0, b
    if kind == "box300x800":                              # length != width: x and y are both tested against width
        b = np.zeros((20, 5))
        b[:, 0] = rng.uniform(0, 300, 20); b[:, 1] = rng.uniform(0, 800, 20)
        b[:, 2] = rng.uniform(1, 5, 20); b[:, 3] = rng.uniform(5, 25, 20); b[:, 4] = rng.uniform(10, 120, 20)
        return 300.0, 800.0, 80.0, b
    if kind == "apf":
        # 56 wide, flat discs (R 30, H 3) stacked on the centre plus 8 others: 10 m above them the 3-D distance to every disc
        # centre is inside its radius, so UAV.cal_force passes 100 within those 56 obstacles (the early return)
        b = np.zeros((64, 5))
        b[:56, 0] = 250 + rng.uniform(-6, 6, 56); b[:56, 1] = 250 + rng.uniform(-6, 6, 56)
        b[:56, 2] = 0.0; b[:56, 3] = 30.0; b[:56, 4] = 3.0
        b[56:, 0] = rng.uniform(50, 450, 8); b[56:, 1] = rng.uniform(50, 450, 8)
        b[56:, 2] = 2.0; b[56:, 3] = rng.uniform(5, 15, 8); b[56:, 4] = rng.uniform(20, 90, 8)
        return 500.0, 500.0, 100.0, b
    raise KeyError(kind)


CITIES = ("empty", "one", "dense64", "box300x800", "apf")


def cities(kind, seed=0):
    from uavrl_b200 import engine
    L, W, H, b = make_city(kind, seed)
    return engine.City(L, W, H, b), O.OracleCity(L, W, H, b)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def small_batch_envs():
    """env.cuh small_batch_envs(): 4 CTAs of 8 envs per SM.  N <= this runs env_kernel<true, 8>, N above it
    env_kernel<true, 32> (env.cu launch_env_step); with extras it is always the 8-env instance."""
    return 4 * sm_count() * 8


# ----------------------------------------------------------------------------------------------------------- pools
def hand_pool(ocity, P, K, rng, n_sub=None, alias=None, z=(2.0, 40.0), near=None):
    """Start / goal / straight sub-goal paths of n_sub entries (default 1..K), starts outside every threat (a quarter of
    them within near = (x, y, r) when given)."""
    W, Hh = ocity.c.width, ocity.c.h
    start = np.zeros((P, 3))
    for i in range(P):
        lo, hi = (3, 3, z[0]), (W - 3, W - 3, min(z[1], Hh - 1))
        if near is not None and i % 4 == 0:
            lo, hi = (near[0] - near[2], near[1] - near[2], z[0]), (near[0] + near[2], near[1] + near[2], min(z[1], Hh - 1))
        while True:
            q = rng.uniform(lo, hi)
            if ocity.threaten_rate(q)[0] == 0:
                start[i] = q
                break
    goal = rng.uniform((3, 3, 0), (W - 3, W - 3, min(z[1], Hh - 1)), (P, 3))
    ns = rng.integers(1, K + 1, P) if n_sub is None else np.broadcast_to(np.asarray(n_sub, np.int32), (P,)).copy()
    al = rng.integers(0, 2, P).astype(np.uint8) if alias is None else np.full(P, alias, np.uint8)
    sub = np.zeros((P, K, 3))
    for i in range(P):
        n = int(ns[i])
        f = np.arange(n) / max(n - 1, 1)
        sub[i, :n] = start[i] + f[:, None] * (goal[i] - start[i])
        if n > 1:
            sub[i, 1:n - 1] += rng.normal(0, 2, (n - 2, 3)) * (1, 1, 0.2)
        if not al[i]:
            sub[i, 0] += (rng.normal(0, 3), rng.normal(0, 3), 0.0)
        sub[i, n - 1] = goal[i]
    return dict(start=start, goal=goal, heading=rng.uniform(0, 2 * np.pi, P), sub=sub, n_sub=ns.astype(np.int32), alias0=al)


def oracle_auto_reset(ob, sc, scen, N, P, ocity, oparams, K):
    """UAV.reset() at the episode boundary, oracle side: an ended env restarts from scenario (scen + N) mod P."""
    ended = np.nonzero(ob.done)[0]
    if ended.size:
        scen[ended] = (scen[ended] + N) % P
        s = scen[ended]
        fresh = O.OracleBatch(ocity, oparams, ended.size, K)
        fresh.reset(sc["start"][s], sc["goal"][s], sc["heading"][s], sc["sub"][s], sc["n_sub"][s], sc["alias0"][s])
        for k in F64 + ("step", "cursor", "n_sub", "done", "alias0"):
            getattr(ob, k)[ended] = getattr(fresh, k)
        ob.goal[ended] = fresh.goal; ob.sub[ended] = fresh.sub
    return ended.size


def assert_obs_heading_on_circle(got, want64, what):
    """assert_obs with obs[7] (calculate_angle(0, V_vector)) compared on the circle, and inside [0, 2 pi].  The greedy f64
    actions of seek() cancel the heading to the last bit, so the new heading lands within ulps of 0 = 2 pi; the cached
    heading and the reference's degree round trip of the previous one differ by ulps and may end on opposite sides of the
    wrap (0 against 6.283: the same direction; positions and rewards agree)."""
    got = np.array(got); want64 = np.array(want64, np.float64)
    h, hw = got[:, 7].astype(np.float64), want64[:, 7]
    assert ((h >= 0) & (h <= np.float32(2 * np.pi))).all(), (what, "obs[7] outside [0, 2 pi]")
    d = np.abs(h - hw)
    assert (np.minimum(d, 2 * np.pi - d) <= 1e-5 * np.maximum(1.0, hw) + 1e-5).all(), (what, "obs[7]")
    got[:, 7] = 0; want64[:, 7] = 0
    assert_obs(got, want64, what)


def seek(ob, params, rng, kind, bound):
    """Half the envs steer toward their sub-goal (so that pops and successes happen), the rest act at random."""
    N = ob.n
    e = np.arange(N)
    c = np.minimum(ob.cursor, ob.kmax - 1)
    sg = ob.sub[e, c]
    sg = np.where((ob.alias0.astype(bool) & (ob.cursor == 0))[:, None], np.stack([ob.px, ob.py, ob.pz], 1), sg)
    want = np.arctan2(sg[:, 1] - ob.py, sg[:, 0] - ob.px)
    have = np.arctan2(ob.vy, ob.vx)
    d = (want - have + np.pi) % (2 * np.pi) - np.pi
    greedy = rng.uniform(size=N) < 0.5
    if kind == "d27":
        i = np.clip(np.round(d / params.steering), -1, 1).astype(np.int32) + 1
        j = np.where(sg[:, 2] > ob.pz + 0.5, 2, np.where(sg[:, 2] < ob.pz - 0.5, 0, 1))
        a = i * 9 + j * 3 + rng.integers(0, 3, N)
        return np.where(greedy, a, rng.integers(0, 27, N)).astype(np.int32)
    a = np.clip(d / params.steering, -bound, bound)
    return np.where(greedy, a, rng.uniform(-bound, bound, N))


KIND = {"d27": ("ACT_DISCRETE27", torch.int32), "f64": ("ACT_CONT_F64", torch.float64),
        "f32": ("ACT_CONT_F32", torch.float32), "f32x2": ("ACT_CONT_F32X2", torch.float32)}


POWER = dict(P_i=89.0, v_0=4.05, d_0=0.6, rho=1.225, s=0.05, A=0.53, P_b=79.0, F_b=120.0, xi=0.82)


def fly_power(V):
    return O.lib().ora_fly_power(float(V), *[POWER[k] for k in ("P_i", "v_0", "d_0", "rho", "s", "A", "P_b", "F_b", "xi")])


SHIPPED = dict(max_v=1.0, min_v=0.6, steering=np.pi / 6, climb_rate=1.0, max_step=150)


def params_of(**kw):
    d = dict(SHIPPED)
    d.update(kw)
    return d
