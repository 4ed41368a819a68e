"""Moving-obstacle sweep: the optional-model env step (env_extras_kernel) with a moving table, against the CPU oracle on the same
table rule (motion_oracle.MovingCity), across non-square boxes, wall-bound and fast tables, every extra, every action kind,
sub-goal capacities and batch sizes.  Each row runs engine.EnvBatch with set_motion and oracle.OracleBatch side by side with
the tolerances of the env sweep (test_env_shapes_gpu.py): every integer output exact, fp64 state and reward 1e-9 relative, the
observation with its heading on the circle, the APF queues, energy, tracked paths and episode records, and env.obstacles()
bit for bit against the Python rule.  One oracle-free check runs on every step: the observation's 80 occupancy bits equal
threaten_rate (threat_kernel: every cylinder, no cull) at the probe points on the current table, which checks the step's
candidate mask and its widening by the table's reach.  Each row asserts the branches it exists for with counters.

The other tests place a cylinder just beyond the static cull reach and move it into a probe window (test_cull_reach), observe
after set_state on a moved table, test the refusal bounds of set_motion on non-square boxes at the boundary, the table's
lifecycle, threaten_rate next to every moved boundary, and episode records and evaluation under motion."""
import zlib

import numpy as np
import pytest
import torch

import motion_oracle as MO
import oracle as O
from env_sweep import (F64, KIND, POWER, assert_obs_heading_on_circle, fly_power, hand_pool, make_city, oracle_auto_reset,
                       params_of, seek)
from gpu_util import MAX_STEP, assert_close64, assert_obs, assert_same, learner, sac, short_episode_env
from uavrl_b200 import _lib, engine

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- tables
def motion_city(kind, seed=0):
    """(len, width, h, buildings [n, 5], velocity [n, 3]) of a moving city: centres inside [0, len] x [0, width]."""
    rng = np.random.default_rng(seed + 101)
    if kind == "one":
        L, W, H, b = make_city("one")
        return L, W, H, b, np.array([[3.75, -2.5, 0.0]])
    if kind == "dense64c":                                # dense64 with the centres straddling the box clamped into it
        L, W, H, b = make_city("dense64")
        b = b.copy()
        b[:, 0] = np.clip(b[:, 0], 0.0, L); b[:, 1] = np.clip(b[:, 1], 0.0, W)
        v = np.zeros((64, 3)); v[:, :2] = rng.normal(0, 2.5, (64, 2)); v[::5] = 0.0; v[1::7, 2] = 0.25
        return L, W, H, b, v
    if kind in ("box300x800", "box800x300"):
        L, W, H, b = make_city("box300x800")
        b = b.copy()
        if kind == "box800x300":                          # the same cylinders mirrored: len 800 > width 300
            L, W = W, L
            b[:, [0, 1]] = b[:, [1, 0]]
        v = np.zeros((20, 3)); v[:, 0] = rng.normal(0, 6, 20); v[:, 1] = rng.normal(0, 6, 20)
        v[0, 0] = L; v[1, 1] = -W; v[2, :2] = (-L, W)     # |vx| = len (> width on 800 x 300), |vy| = width
        return L, W, H, b, v
    if kind == "apf":                                     # the 56-disc stack drifts slowly: cum > 100 stays reachable
        L, W, H, b = make_city("apf")
        v = np.zeros((64, 3)); v[:56, :2] = rng.normal(0, 0.15, (56, 2)); v[56:, :2] = rng.normal(0, 1.5, (8, 2))
        return L, W, H, b, v
    if kind == "walls":                                   # centres on the walls and corners, some bouncing wall to wall
        L, W, H = 400.0, 600.0, 100.0
        b = np.zeros((24, 5))
        b[:, 0] = rng.uniform(0, L, 24); b[:, 1] = rng.uniform(0, W, 24)
        b[:4, 0] = 0.0; b[4:8, 0] = L; b[8:12, 1] = 0.0; b[12:16, 1] = W
        b[16:20, :2] = [(0.0, 0.0), (L, 0.0), (0.0, W), (L, W)]
        b[:, 2] = 0.0; b[:, 3] = rng.uniform(8, 25, 24); b[:, 4] = rng.uniform(15, 90, 24)
        v = np.zeros((24, 3)); v[:, :2] = rng.normal(0, 8, (24, 2))
        v[0:24:3, 0] = L * np.sign(rng.normal(size=8)); v[1:24:3, 1] = W * np.sign(rng.normal(size=8))
        v[0, 0] = L; v[9, 1] = W                          # from x = 0 (y = 0) onto x = len (y = width): not a reflection
        v[20] = 0.0
        return L, W, H, b, v
    if kind == "fast":
        # 20-60 m per step on each axis; a third are wide, flat discs, so that a UAV flying over one is inside its 3-D radius
        # without a collision: UAV.cal_force pushes the aliased sub-goal off the start by more than the 7 m radius
        L, W, H = 500.0, 500.0, 100.0
        b = np.zeros((40, 5))
        b[:, 0] = rng.uniform(0, L, 40); b[:, 1] = rng.uniform(0, W, 40)
        b[:, 2] = 0.0; b[:, 3] = rng.uniform(10, 25, 40); b[:, 4] = rng.uniform(20, 80, 40)
        b[::3, 3] = rng.uniform(25, 35, 14); b[::3, 4] = rng.uniform(1.0, 3.0, 14)
        v = np.zeros((40, 3)); v[:, :2] = rng.uniform(20, 60, (40, 2)) * rng.choice([-1.0, 1.0], (40, 2))
        return L, W, H, b, v
    raise KeyError(kind)


MOTION_CITIES = ("one", "dense64c", "box300x800", "box800x300", "apf", "walls", "fast")


def table_of(b, v):
    tab = np.zeros((b.shape[0], 4))
    tab[:, :2] = b[:, :2]; tab[:, 2:] = v[:, :2]
    return tab


def assert_table(env, tab, what):
    pos, vel, _ = env.obstacles()
    assert np.array_equal(pos[:, :2], tab[:, :2]) and np.array_equal(vel[:, :2], tab[:, 2:]), what


def probe_bits(env, st):
    """threaten_rate at every env's 80 probe points on the current table -> [n, 80] in PROBE_SLOT order."""
    pts = MO.probe_points(st["px"], st["py"], st["pz"])
    return env.threaten_rate(pts.reshape(-1, 3)).reshape(-1, 80)


def probe_hits(pts, tab, b):
    """[n, 80, nc]: probe point inside a cylinder of the table (building.check_threaten, with R and H of b), in numpy"""
    dx = pts[:, :, 0, None] - tab[None, None, :, 0]
    dy = pts[:, :, 1, None] - tab[None, None, :, 1]
    return (pts[:, :, 2, None] <= b[None, None, :, 4]) & (np.sqrt(dx * dx + dy * dy) < b[None, None, :, 3])


# ----------------------------------------------------------------------------------------------------------- the row runner
def run_motion_row(city_kind, N, K, params_kw, kind="d27", T=40, ext=(), pool_kw=None, age=(None, None), seed=0):
    """Step the CUDA env with a moving table and the oracle on MovingCity side by side; returns counters."""
    L, W, H, b, vel = motion_city(city_kind)
    apf, energy, records = "apf" in ext, "energy" in ext, "records" in ext
    params, oparams = engine.UavParams(**params_kw), O.UavParams(**params_kw)
    rng = np.random.default_rng(seed)
    static = O.OracleCity(L, W, H, b)
    P = max(2 * N, 16) if N < 4096 else N + 64
    sc = hand_pool(static, P, K, rng, **(pool_kw or {}))
    env = engine.EnvBatch(engine.City(L, W, H, b), params, N, max_subgoals=K, auto_reset=True)
    mc = MO.MovingCity(L, W, H, b, table_of(b, vel), vel[:, 2], apf=apf)
    track = min(N, 8) if energy else 0
    try:
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
        xkw = dict(power=POWER, track_envs=track, track_capacity=64) if energy else {}
        if apf:
            xkw["obstacle_v"] = vel
        if xkw:
            env.set_extras(**xkw)
        env.set_motion(vel, positions=b[:, :3])
        if records:
            env.set_records(N * (T + 1))
        env.reset(0)
        scen = np.arange(N) % P
        ob = O.OracleBatch(mc.city, oparams, N, K)
        ob.reset(sc["start"][scen], sc["goal"][scen], sc["heading"][scen], sc["sub"][scen], sc["n_sub"][scen], sc["alias0"][scen])
        assert_obs(env.observe().cpu().numpy(), ob.state(want64=True)[1], "obs0")
        assert_table(env, mc.tab, "observe advanced the table")
        cnt = dict(coll=0, moved_coll=0, pop=0, lose=0, success=0, restart=0, cull=0, alias_kept_coll=0, alias_kept_free=0,
                   records=0, x0=0, xlen=0, y0=0, ywidth=0)
        kname, tdt = KIND[kind]
        static_reach = b[:, 3] + 20.0 + params_kw["max_v"] + 0.5
        en = np.zeros(N)
        ep_steps = np.zeros(N, np.int64); ep_coll = np.zeros(N, np.int64); ordinal = np.zeros(N, np.int64)
        want_rec = {}
        for t in range(T):
            w = "t%d" % t
            pre = np.stack([ob.px, ob.py, ob.pz], 1)
            tab_t = mc.tab.copy()
            alias_first = ob.alias0.astype(bool) & (ob.cursor == 0)
            a = seek(ob, oparams, rng, kind, 1.0)
            if kind == "f32x2":
                a2 = np.stack([a.astype(np.float32), rng.uniform(-9, 9, N).astype(np.float32)], 1)    # only [.., 0] steers
                act, a64 = torch.tensor(a2, device="cuda"), a2[:, 0].astype(np.float64)
            elif kind == "f32":
                act, a64 = torch.tensor(a.astype(np.float32), device="cuda"), a.astype(np.float32).astype(np.float64)
            else:
                act, a64 = torch.tensor(a, dtype=tdt, device="cuda"), a.astype(np.float64)
            cur_before = ob.cursor.copy()
            out = env.step(act, kind=getattr(_lib, kname))
            rew, done, info, coll, _ = ob.step_(a64, O.ACT_DISCRETE27 if kind == "d27" else O.ACT_CONTINUOUS, want_obs=False)
            mc.advance()
            o = {k: v.cpu().numpy() for k, v in out.items()}
            assert np.array_equal(o["done"], done) and np.array_equal(o["info"], info), w
            assert np.array_equal(o["collision"], coll) and np.array_equal(o["ended"], ob.done), w
            np.testing.assert_allclose(o["reward"], rew, rtol=1e-5, atol=1e-5)
            st = env.get_state()
            assert_close64(st["reward64"], rew, 1e-9, "reward " + w)
            # a collision where the cylinders as created leave the attempted point free: a moved cylinder caused it
            dz = ((a64.astype(np.int64) // 3) % 3 - 1) * params_kw["climb_rate"] if kind == "d27" else np.zeros(N)
            tried = np.stack([pre[:, 0] + ob.vx, pre[:, 1] + ob.vy, pre[:, 2] + dz], 1)
            hit = np.nonzero(coll)[0]
            if hit.size:
                cnt["moved_coll"] += int((static.threaten_rate(tried[hit]) == 0).sum())
            ended = ob.done.astype(bool).copy()
            kept = alias_first & (ob.cursor == 0) & ~ended
            cnt["alias_kept_coll"] += int((kept & (coll == 1)).sum()); cnt["alias_kept_free"] += int((kept & (coll == 0)).sum())
            if energy:
                en = en + np.array([fly_power(v) for v in ob.V])
                got_en = env.get_energy()
                np.testing.assert_allclose(got_en[~ended], en[~ended], rtol=1e-12, atol=1e-9)
                assert (got_en[ended] == 0).all(), w                # an ended env restarts with 0
            ep_steps += 1; ep_coll += coll
            end_pos = np.stack([ob.px, ob.py, ob.pz], 1)
            for e in np.nonzero(ended)[0]:
                if records:
                    s = int(scen[e])
                    want_rec[int(ordinal[e] * N + e)] = dict(
                        scenario=s, env=e, ordinal=int(ordinal[e]), outcome=int(info[e]), steps=int(ep_steps[e]),
                        subgoals=int(ob.cursor[e]), collisions=int(ep_coll[e]), total_score=ob.total_score[e], path_len=ob.path_len[e],
                        final_dist=float(np.linalg.norm(end_pos[e] - ob.goal[e])), energy=en[e] if energy else 0.0)
                ordinal[e] += 1
            ep_steps[ended] = 0; ep_coll[ended] = 0; en[ended] = 0.0
            cnt["pop"] += int(((ob.cursor > cur_before) & (info == 1)).sum())
            cnt["restart"] += oracle_auto_reset(ob, sc, scen, N, P, mc.city, oparams, K)
            assert np.array_equal(st["scenario"], scen), w
            assert np.array_equal(st["step"], ob.step) and np.array_equal(st["cursor"], ob.cursor), w
            assert np.array_equal(st["done"], ob.done), w
            for k in F64:
                assert_close64(st[k], getattr(ob, k), 1e-9, k + " " + w)
            assert_obs_heading_on_circle(o["obs"], ob.state(want64=True)[1], "obs " + w)
            bits = probe_bits(env, st)
            assert np.array_equal(o["obs"][:, MO.PROBE_SLOT], bits.astype(np.float32)), ("probe bits vs threaten_rate", w)
            if N <= 2048:
                # cull entries: a cylinder some probe of the env hits on O_{t+1} whose O_t centre was beyond the static cull
                # reach of the point the step culled from (the pre-step position, or the restart position)
                cpos = np.where(ended[:, None], np.stack([ob.px, ob.py], 1), pre[:, :2])
                far = (np.abs(cpos[:, None, 0] - tab_t[None, :, 0]) > static_reach) | (np.abs(cpos[:, None, 1] - tab_t[None, :, 1]) > static_reach)
                seen = probe_hits(MO.probe_points(st["px"], st["py"], st["pz"]), mc.tab, b).any(1)
                cnt["cull"] += int((far & seen).sum())
            if apf:
                subs = env.get_subgoals()
                for e in range(0, N, 1 if N <= 256 else max(1, N // 64)):
                    c, n = int(ob.cursor[e]), int(ob.n_sub[e])
                    assert_close64(subs[e, c:n], ob.sub[e, c:n], 1e-9, "queue e%d %s" % (e, w))
                ob.sub[:] = subs                          # the oracle continues from the kernel's queues
            for e in range(track):                        # UAV.path: the position after every step of the episode
                path = env.get_path(e, 1 if ended[e] else 0)
                assert len(path) >= 1, (e, w)
                assert_close64(path[-1], end_pos[e], 1e-9, "path e%d %s" % (e, w))
            assert_table(env, mc.tab, "table " + w)
            assert env.obstacles()[2] == t + 1
            for k, v in MO.wall_reflections(tab_t, mc.tab).items():
                cnt[k] += v
            cnt["coll"] += int(coll.sum()); cnt["lose"] += int((info == 2).sum()); cnt["success"] += int((info == 1).sum())
            if t == 0 and age[0] is not None:
                aged = rng.integers(age[0], age[1], N).astype(np.int32)
                env.set_state(step=aged); ob.step[:] = aged
        if records:
            rec = env.records(clear=False)
            assert sorted(want_rec) == list(rec["slot"]) and rec["n_dropped"] == 0
            for i, slot in enumerate(rec["slot"]):
                wr = want_rec[int(slot)]
                for k in ("scenario", "env", "ordinal", "outcome", "steps", "subgoals", "collisions"):
                    assert int(rec[k][i]) == wr[k], (k, int(slot))
                for k in ("total_score", "path_len", "final_dist", "energy"):
                    assert_close64(rec[k][i], wr[k], 1e-9, "record %s slot %d" % (k, slot))
            cnt["records"] = len(want_rec)
        if city_kind == "apf":                            # UAV.cal_force's cum > 100 return stays reachable on the moved stack
            d = np.sqrt((mc.tab[:, 0] - 250) ** 2 + (mc.tab[:, 1] - 250) ** 2 + (10 - b[:, 2]) ** 2) - b[:, 3]
            assert (d < 0).sum() > 50
        return cnt
    finally:
        mc.close()
        env.close()


M, MA, ME, MR = ("motion",), ("motion", "apf"), ("motion", "energy"), ("motion", "records")
ALL = ("motion", "apf", "energy", "records")
# id: (city, N, K, params, kind, T, extras, pool_kw, counters that must be > 0)
ROWS = {
    "one_N1_d27": ("one", 1, 8, params_of(max_v=3.0, max_step=30), "d27", 60, M, {"near": (250.0, 250.0, 60.0)},
                   ("lose", "restart")),
    "one_N7_f64_records": ("one", 7, 3, params_of(max_v=3.0, max_step=20), "f64", 60, MR,
                           {"n_sub": 3, "alias": 1, "near": (250.0, 250.0, 60.0)}, ("coll", "moved_coll", "lose", "records")),
    "dense64c_N257_d27_apf": ("dense64c", 257, 8, params_of(max_v=2.0, max_step=30), "d27", 40, MA, {"z": (1.0, 30.0)},
                              ("coll", "moved_coll", "pop", "lose", "restart", "cull")),
    "dense64c_N16395_d27_energy": ("dense64c", 16395, 8, params_of(max_v=3.0, min_v=1.0, max_step=30), "d27", 10, ME,
                                   {"z": (1.0, 30.0)}, ("coll", "lose", "restart")),
    "box300x800_N8_f32_energy": ("box300x800", 8, 2, params_of(max_v=3.0, min_v=1.0, max_step=20), "f32", 50, ME,
                                 {"n_sub": 2, "alias": 0}, ("lose", "restart")),
    "box300x800_N33_d27_all": ("box300x800", 33, 3, params_of(max_v=3.0, max_step=20), "d27", 50, ALL,
                               {"n_sub": 3, "alias": 1}, ("coll", "lose", "restart", "records", "x0", "xlen", "y0", "ywidth")),
    "box800x300_N9_f32x2_records": ("box800x300", 9, 3, params_of(max_v=3.0, max_step=20), "f32x2", 50, MR,
                                    {"n_sub": 3, "alias": 0}, ("lose", "restart", "records", "x0", "xlen", "y0", "ywidth")),
    "box800x300_N257_d27_apf": ("box800x300", 257, 2, params_of(max_v=3.0, max_step=20), "d27", 40, MA,
                                {"n_sub": 2, "alias": 1}, ("coll", "moved_coll", "pop", "lose", "restart")),
    "apf_N33_d27_all": ("apf", 33, 8, params_of(max_v=3.0, max_step=30), "d27", 30, ALL,
                        {"z": (8.0, 14.0), "near": (250.0, 250.0, 12.0), "alias": 0}, ("coll", "pop", "lose", "records")),
    "walls_N257_d27": ("walls", 257, 8, params_of(max_v=3.0, max_step=30), "d27", 40, M, {"z": (1.0, 40.0)},
                       ("coll", "moved_coll", "lose", "restart", "cull", "x0", "xlen", "y0", "ywidth")),
    "walls_N9_f64_all": ("walls", 9, 1, params_of(max_v=3.0, max_step=20), "f64", 50, ALL, {"n_sub": 1},
                         ("lose", "restart", "records", "x0", "xlen", "y0", "ywidth")),
    "fast_N257_d27_apf_alias": ("fast", 257, 2, params_of(max_v=2.0, max_step=6), "d27", 50, MA,
                                {"n_sub": 2, "alias": 1, "z": (1.0, 12.0)},
                                ("coll", "moved_coll", "lose", "restart", "cull", "alias_kept_coll", "alias_kept_free")),
    "fast_N33_f64_all_K1": ("fast", 33, 1, params_of(max_v=3.0, max_step=20), "f64", 40, ALL, {"n_sub": 1},
                            ("coll", "moved_coll", "success", "restart", "records", "cull")),
    "fast_N8_f32x2_energy_K3": ("fast", 8, 3, params_of(max_v=3.0, max_step=20), "f32x2", 40, ME, {"n_sub": 3, "alias": 0},
                                ("coll", "moved_coll", "lose", "cull")),
}


@pytest.mark.parametrize("row", sorted(ROWS))
def test_motion_row_against_oracle(row):
    city, N, K, params, kind, T, ext, pool_kw, need = ROWS[row]
    age = (max(0, params["max_step"] - 8), params["max_step"]) if params["max_step"] > 8 else (None, None)
    cnt = run_motion_row(city, N, K, params, kind=kind, T=T, ext=ext, pool_kw=pool_kw, age=age, seed=zlib.crc32(row.encode()) % 1000)
    for k in need:
        assert cnt[k] > 0, (row, k, cnt)


# ----------------------------------------------------------------------------------------------------------- cull reach
def test_cull_reach():
    """One cylinder placed 1 ulp to 0.5 m beyond the static cull reach R + 20 + max_v + 0.5 of a UAV heading away from it, moving
    toward the UAV at 0.6, 3, 19.9, 45 m per step and at len / width (arriving by a reflection off the far wall), along each
    axis and diagonal: after one step the occupancy bits equal threaten_rate on the moved table and the oracle, and the
    cylinder is seen wherever the geometry puts it inside a probe window.  Without the cull's widening by the table's reach
    the kernel misses it."""
    L, W, H = 300.0, 500.0, 100.0                         # cylinders in x <= 300; the UAV's box is [0, 500]^2 (y's width)
    R, max_v = 10.0, 0.02
    reach = R + 20.0 + max_v + 0.5
    params = params_of(max_v=max_v, min_v=0.0, max_step=50)
    seen_n = total = 0
    for s in (0.6, 3.0, 19.9, 45.0, "len"):
        for d in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (1, -1), (-1, 1), (-1, -1)):
            for delta in (("ulp", 0.5) if s != "len" else ("far",)):
                c = np.zeros(2)
                if s == "len":
                    # |v| = len / width: the cylinder crosses the box, reflects off the far wall (x + vx leaves [0, box] on
                    # either side, x' = box - x) and lands off = 29 m (axis) / 25 m (diagonal) from the UAV on each moving axis
                    u = np.array([250.0, 400.0, 5.0])
                    off = 29.0 if 0 in d else 25.0
                    for ax in (0, 1):
                        c[ax] = u[ax] if d[ax] == 0 else (L, W)[ax] - (u[ax] + d[ax] * off)
                    v = np.array([L * d[0], W * d[1], 0.0])
                else:
                    u = np.array([150.0, 250.0, 5.0])
                    for ax in (0, 1):
                        edge = u[ax] - d[ax] * reach
                        c[ax] = u[ax] if d[ax] == 0 else np.nextafter(edge, edge - d[ax]) if delta == "ulp" else edge - d[ax] * 0.5
                    v = np.array([s * d[0], s * d[1], 0.0])
                assert 0 <= c[0] <= L and 0 <= c[1] <= W
                b = np.array([[c[0], c[1], 0.0, R, 40.0]])
                env = engine.EnvBatch(engine.City(L, W, H, b), engine.UavParams(**params), 1, max_subgoals=2)
                mc = MO.MovingCity(L, W, H, b, table_of(b, v[None]), 0.0)
                try:
                    g = u + np.array([-80.0 * np.sign(d[0] or 0.1), -80.0 * np.sign(d[1] or 0.1), 0.0])
                    env.set_pool(u[None], g[None], [0.0], np.stack([u, g])[None], [2], [0])
                    env.set_motion(v[None], positions=b[:, :3])
                    env.set_records(4)                    # records on: the extras step without any other model
                    env.reset(0)
                    hv = -np.array([np.sign(d[0]), np.sign(d[1])], np.float64)     # heading away from the cylinder
                    hv = hv / max(np.hypot(*hv), 1e-300) * max_v
                    env.set_state(px=u[:1], py=u[1:2], pz=u[2:], vx=hv[:1], vy=hv[1:], V=[np.hypot(*hv)])
                    ob = O.OracleBatch(mc.city, O.UavParams(**params), 1, 2)
                    ob.reset(u[None], g[None], [0.0], np.stack([u, g])[None], [2], [0])
                    for k, x in (("px", u[0]), ("py", u[1]), ("pz", u[2]), ("vx", hv[0]), ("vy", hv[1]), ("V", np.hypot(*hv))):
                        getattr(ob, k)[:] = x
                    out = env.step(torch.zeros(1, dtype=torch.float64, device="cuda"), kind=_lib.ACT_CONT_F64)
                    MO.step(mc, ob, [0.0], O.ACT_CONTINUOUS)
                    obs = out["obs"].cpu().numpy()
                    st = env.get_state()
                    bits = probe_bits(env, st)
                    what = (s, d, delta)
                    assert_table(env, mc.tab, what)
                    assert np.array_equal(obs[:, MO.PROBE_SLOT], bits.astype(np.float32)), what
                    assert_obs(obs, ob.state(want64=True)[1], str(what))
                    far = max(abs(u[0] - c[0]), abs(u[1] - c[1])) > reach
                    assert far, what
                    seen = probe_hits(MO.probe_points(st["px"], st["py"], st["pz"]), mc.tab, b).any()
                    assert bool(bits.any()) == bool(seen), what
                    seen_n += int(seen); total += 1
                    if s in (19.9, 45.0, "len") or (s == 3.0 and 0 in d) or (s == 0.6 and 0 in d and delta == "ulp"):
                        assert seen, what
                finally:
                    mc.close()
                    env.close()
    assert total == 72 and seen_n >= 44, (total, seen_n)


# ----------------------------------------------------------------------------------------------------------- observe
@pytest.mark.parametrize("city", MOTION_CITIES)
@pytest.mark.parametrize("k", [1, 7])
def test_observe_after_set_state_moved(city, k):
    """observe() with the optional models on (env_extras_kernel<false, 32>) after k steps of the table and set_state at random
    positions, points 19.5 / 20 m from each box edge and zero and signed-zero velocities, at N = 1, 31, 33, 333 (ragged last
    CTAs): against the oracle on the same table, and observe() leaves the table where it is."""
    L, W, H, b, vel = motion_city(city)
    params = params_of(max_v=3.0)
    K = 4
    static = O.OracleCity(L, W, H, b)
    for N in (1, 31, 33, 333):
        rng = np.random.default_rng(N + 10 * k)
        sc = hand_pool(static, N, K, rng)
        env = engine.EnvBatch(engine.City(L, W, H, b), engine.UavParams(**params), N, max_subgoals=K)
        mc = MO.MovingCity(L, W, H, b, table_of(b, vel), vel[:, 2])
        try:
            env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
            env.set_motion(vel, positions=b[:, :3])
            env.reset(0)
            for _ in range(k):
                env.step(torch.full((N,), 13, dtype=torch.int32, device="cuda"))
                mc.advance()
            assert_table(env, mc.tab, "table after %d steps" % k)
            env.reset(0)                                  # cursors and flags as the oracle's; the table stays
            ob = O.OracleBatch(mc.city, O.UavParams(**params), N, K)
            ob.reset(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
            px = rng.uniform(-2, W + 2, N); py = rng.uniform(-2, W + 2, N); pz = rng.uniform(-1, H + 1, N)
            edges = [0.0, W, 19.5, W - 19.5, 20.0, W - 20.0]
            px[:min(N, 12)] = rng.choice(edges, min(N, 12)); py[:min(N, 6)] = rng.choice(edges, min(N, 6))
            # and next to the moved cylinders
            near = rng.integers(0, b.shape[0], N)
            sel = np.arange(N) % 3 == 2
            px[sel] = mc.tab[near[sel], 0] + rng.uniform(-30, 30, sel.sum()); py[sel] = mc.tab[near[sel], 1] + rng.uniform(-30, 30, sel.sum())
            pz[sel] = rng.uniform(0, 30, sel.sum())
            vx = rng.uniform(-3, 3, N); vy = rng.uniform(-3, 3, N)
            z = np.arange(N) % 5 == 1
            vx[z] = rng.choice([0.0, -0.0], z.sum()); vy[z] = rng.choice([0.0, -0.0], z.sum())
            V = np.hypot(vx, vy)
            step = rng.integers(0, 150, N).astype(np.int32)
            env.set_state(px=px, py=py, pz=pz, vx=vx, vy=vy, V=V, step=step)
            for key, val in (("px", px), ("py", py), ("pz", pz), ("vx", vx), ("vy", vy), ("V", V), ("step", step)):
                getattr(ob, key)[:] = val
            got = env.observe().cpu().numpy()
            assert_obs(got, ob.state(want64=True)[1], "%s k%d N%d" % (city, k, N))
            assert np.array_equal(got[:, MO.PROBE_SLOT], probe_bits(env, env.get_state()).astype(np.float32))
            assert_table(env, mc.tab, "observe advanced the table")
            assert env.obstacles()[2] == k
        finally:
            mc.close()
            env.close()


# ----------------------------------------------------------------------------------------------------------- refusals
def up(v):
    return np.nextafter(v, np.inf)


def dn(v):
    return np.nextafter(v, -np.inf)


@pytest.mark.parametrize("box", ["box300x800", "box800x300"])
def test_refusal_bounds_on_non_square_boxes(box):
    """set_motion on a non-square box: x = len, y = width, x = -0.0, |vx| = len (above width when len > width) and |vy| = width
    are accepted, one ulp beyond each is refused, and every refusal leaves obstacles(), get_state() and get_subgoals() as they
    were."""
    L, W, H, b, vel = motion_city(box)
    env = engine.EnvBatch(engine.City(L, W, H, b), engine.UavParams(**params_of(max_v=2.0)), 16, max_subgoals=4, auto_reset=True)
    try:
        sc = hand_pool(O.OracleCity(L, W, H, b), 32, 4, np.random.default_rng(1))
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
        env.set_extras(obstacle_v=vel)
        env.set_motion(vel, positions=b[:, :3])
        env.reset(0)
        for _ in range(3):
            env.step(torch.zeros(16, dtype=torch.int32, device="cuda"))

        def snap():
            return env.obstacles(), env.get_state(), env.get_subgoals()

        def same(x, y):
            assert all(np.array_equal(p, q) for p, q in zip(x[0], y[0]))
            assert all(np.array_equal(x[1][k], y[1][k]) for k in x[1]) and np.array_equal(x[2], y[2])

        env.set_extras()                                  # APF off: the velocities below need not match obstacle_v
        env.reset(0)
        pos = b[:, :3].copy()
        ok = []
        for row, col, val in ((0, 0, L), (1, 1, W), (2, 0, -0.0), (3, 1, -0.0), (4, 0, 0.0)):
            p = pos.copy(); p[row, col] = val
            ok.append(dict(velocity=vel, positions=p))
        for row, col, val in ((0, 0, L), (1, 0, -L), (2, 1, W), (3, 1, -W)):
            v = vel.copy(); v[row, col] = val
            ok.append(dict(velocity=v, positions=pos))
        bad = []
        for row, col, val in ((0, 0, up(L)), (1, 1, up(W)), (2, 0, dn(-0.0)), (3, 1, dn(0.0))):
            p = pos.copy(); p[row, col] = val
            bad.append(dict(velocity=vel, positions=p))
        for row, col, val in ((0, 0, up(L)), (1, 0, dn(-L)), (2, 1, up(W)), (3, 1, dn(-W))):
            v = vel.copy(); v[row, col] = val
            bad.append(dict(velocity=v, positions=pos))
        for kw in ok:
            env.set_motion(**kw)
            pos_got, vel_got, steps = env.obstacles()
            assert steps == 0 and np.array_equal(pos_got[:, :2], kw["positions"][:, :2]) and np.array_equal(vel_got, kw["velocity"])
            env.step(torch.zeros(16, dtype=torch.int32, device="cuda"))
            tab = table_of(np.concatenate([kw["positions"][:, :2], b[:, 2:]], 1), kw["velocity"])
            MO.obstacle_run(tab, L, W)
            assert_table(env, tab, "one run from an accepted boundary row")
        for kw in bad:
            before = snap()
            with pytest.raises(engine.UavrlError):
                env.set_motion(**kw)
            same(before, snap())
    finally:
        env.close()


def test_refusals_of_out_of_box_and_empty_cities():
    """dense64's centres straddling the box edge are refused (the clamped table is what the sweep runs), and a city with no
    cylinders has nothing to move; neither refusal changes the table or the state."""
    L, W, H, b = make_city("dense64")
    env = engine.EnvBatch(engine.City(L, W, H, b), engine.UavParams(**params_of(max_v=2.0)), 8, max_subgoals=4)
    try:
        sc = hand_pool(O.OracleCity(L, W, H, b), 8, 4, np.random.default_rng(2))
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
        env.set_motion(motion_city("dense64c")[4], positions=motion_city("dense64c")[3][:, :3])
        env.reset(0)
        env.step(torch.zeros(8, dtype=torch.int32, device="cuda"))
        before = env.obstacles(), env.get_state()
        for i in range(4):                                # the four straddling rows, one at a time
            p = motion_city("dense64c")[3][:, :3].copy(); p[i] = b[i, :3]
            with pytest.raises(engine.UavrlError, match="outside"):
                env.set_motion(np.zeros((64, 3)), positions=p)
        with pytest.raises(engine.UavrlError, match="outside"):
            env.set_motion(np.zeros((64, 3)), positions=b[:, :3])
        after = env.obstacles(), env.get_state()
        assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0]))
        assert all(np.array_equal(before[1][k], after[1][k]) for k in before[1])
    finally:
        env.close()
    empty = engine.EnvBatch(engine.City(500, 500, 100, np.zeros((0, 5))), engine.UavParams(), 4, max_subgoals=2)
    try:
        with pytest.raises(engine.UavrlError, match="no obstacles"):
            empty.set_motion(np.zeros((0, 3)))
        assert empty.obstacles()[2] == 0
    finally:
        empty.close()


# ----------------------------------------------------------------------------------------------------------- lifecycle
def test_table_lifecycle():
    """reset(), set_pool / generate_pool, set_extras without APF and set_records leave the table and its step count alone;
    set_motion(v) without positions continues from the current centres with steps = 0 and the new velocities; set_motion(None)
    then steps bit for bit like an env that never moved."""
    L, W, H, b, vel = motion_city("box300x800")
    params = engine.UavParams(**params_of(max_v=2.0, max_step=20))
    N = 40

    def make():
        env = engine.EnvBatch(engine.City(L, W, H, b), params, N, max_subgoals=64, auto_reset=True)
        env.generate_pool(128, seed=5)
        return env
    rng = np.random.default_rng(3)
    acts = [torch.tensor(rng.integers(0, 27, N).astype(np.int32), device="cuda") for _ in range(30)]
    env = make()
    try:
        env.set_motion(vel, positions=b[:, :3])
        env.reset(0)
        tab = table_of(b, vel)
        for t in range(5):
            env.step(acts[t]); MO.obstacle_run(tab, L, W)
        assert_table(env, tab, "5 steps")
        for what, fn in (("reset", lambda: env.reset(3)), ("generate_pool", lambda: env.generate_pool(64, seed=9)),
                         ("set_pool", lambda: env.set_pool(*[env.get_pool()[k] for k in ("start", "goal")],
                                                           np.zeros(64), env.get_pool()["sub"], env.get_pool()["n_sub"])),
                         ("set_extras", lambda: env.set_extras(power=POWER, track_envs=2, track_capacity=8)),
                         ("set_records", lambda: env.set_records(64)), ("set_records off", lambda: env.set_records(0))):
            fn()
            assert_table(env, tab, what)
            assert env.obstacles()[2] == 5, what
        env.reset(0)
        v2 = vel.copy(); v2[:, :2] *= -0.5
        env.set_motion(v2)
        tab[:, 2:] = v2[:, :2]
        assert_table(env, tab, "set_motion without positions")
        assert env.obstacles()[2] == 0
        for t in range(5):
            env.step(acts[5 + t]); MO.obstacle_run(tab, L, W)
        assert_table(env, tab, "continued")
        assert env.obstacles()[2] == 5
        env.set_motion(None)
        pos, v, steps = env.obstacles()
        assert steps == 0 and not v.any() and np.array_equal(pos, b[:, :3])
        env.reset(0)
        still = make()                                    # the same pool and extras, never moved
        pool = env.get_pool()
        still.set_pool(pool["start"], pool["goal"], np.zeros(64), pool["sub"], pool["n_sub"])
        still.set_extras(power=POWER, track_envs=2, track_capacity=8)
        still.reset(0)
        for t in range(10, 30):
            oa, ob = env.step(acts[t]), still.step(acts[t])
            for k in oa:
                assert torch.equal(oa[k], ob[k]), (k, t)
        sa, sb = env.get_state(), still.get_state()
        assert all(np.array_equal(sa[k], sb[k]) for k in sa)
        still.close()
    finally:
        env.close()


# ----------------------------------------------------------------------------------------------------------- threaten_rate
def test_threaten_rate_next_to_every_moved_boundary():
    """threaten_rate (threat_kernel on the moving table) on points 1 ulp either side of every moved cylinder's R and H and of
    the box bounds, after some runs on dense64 (clamped) and 300 x 800, against OracleCity.threaten_rate on the moved centres."""
    import math
    rng = np.random.default_rng(4)
    for kind, runs in (("dense64c", 9), ("box300x800", 13)):
        L, W, H, b, vel = motion_city(kind)
        env = engine.EnvBatch(engine.City(L, W, H, b), engine.UavParams(), 4, max_subgoals=2)
        mc = MO.MovingCity(L, W, H, b, table_of(b, vel), vel[:, 2])
        try:
            sc = hand_pool(O.OracleCity(L, W, H, b), 4, 2, rng)
            env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
            env.set_motion(vel, positions=b[:, :3])
            env.reset(0)
            for _ in range(runs):
                env.step(torch.zeros(4, dtype=torch.int32, device="cuda")); mc.advance()
            assert_table(env, mc.tab, kind)
            pts = []
            for (cx, cy), (_, _, _, R, Hc) in zip(mc.tab[:, :2], b):
                for th in rng.uniform(0, 2 * np.pi, 4):
                    x = cx + R * math.cos(th)
                    for xx in (x, up(x), dn(x)):
                        pts.append((xx, cy + R * math.sin(th), min(Hc, H) * 0.5))
                pts += [(cx + R, cy, 1.0), (up(cx + R), cy, 1.0), (dn(cx + R), cy, 1.0), (cx, dn(cy - R), 1.0), (cx, up(cy - R), 1.0)]
                pts += [(cx, cy, Hc), (cx, cy, up(Hc)), (cx, cy, dn(Hc))]
            for v in (0.0, -0.0, up(0.0), dn(0.0), W, up(W), dn(W), L, up(L)):
                pts += [(v, W / 2, 10.0), (W / 2, v, 10.0)]
            for v in (0.0, dn(0.0), H, up(H), dn(H)):
                pts.append((W / 3, 3.0, v))
            pts = np.array(pts)
            got, want = env.threaten_rate(pts), mc.city.threaten_rate(pts)
            assert np.array_equal(got, want), (kind, int((got != want).sum()))
            static = O.OracleCity(L, W, H, b).threaten_rate(pts)
            assert 0 < want.sum() < len(want) and (static != want).any()
            assert env.obstacles()[2] == runs
        finally:
            mc.close()
            env.close()


# ----------------------------------------------------------------------------------------------------------- records and evaluation
FIELDS = list(engine.RECORD_FIELDS)


def dist(a, b):
    """CalMod.Eu_Loc_distance in float64, left to right"""
    d = a - b
    return np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])


def test_record_fields_under_motion():
    """Motion + APF + energy on 300 x 800, no auto-reset, one episode per env driven by step: every record equals what the host
    reads at the ending step (outputs, get_state, get_energy), bit for bit; start2goal and planner_len are the float64
    formulas on the pool."""
    L, W, H, b, vel = motion_city("box300x800")
    N, K = 48, 4
    params = engine.UavParams(**params_of(max_v=3.0, max_step=25))
    sc = hand_pool(O.OracleCity(L, W, H, b), N, K, np.random.default_rng(6), alias=0)
    env = engine.EnvBatch(engine.City(L, W, H, b), params, N, max_subgoals=K)
    try:
        env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"], sc["alias0"])
        env.set_extras(power=POWER, obstacle_v=vel)
        env.set_motion(vel, positions=b[:, :3])
        env.set_records(N)
        env.reset(0)
        rng = np.random.default_rng(7)
        steps = np.zeros(N, np.int64); coll = np.zeros(N, np.int64)
        want = {}
        for t in range(40):
            out = env.step(torch.tensor(rng.integers(0, 27, N).astype(np.int32), device="cuda"))
            ended, info, c = (out[k].cpu().numpy() for k in ("ended", "info", "collision"))
            live = np.array([e not in want for e in range(N)])
            steps[live] += 1; coll[live] += c[live]
            if (ended.astype(bool) & live).any():
                st, en = env.get_state(), env.get_energy()
                for e in np.nonzero(ended.astype(bool) & live)[0]:
                    p, g, s0 = np.array([st["px"][e], st["py"][e], st["pz"][e]]), sc["goal"][e], sc["start"][e]
                    q = sc["sub"][e]
                    plen = 0.0
                    for i in range(1, int(sc["n_sub"][e])):
                        plen = plen + float(dist(q[i - 1], q[i]))
                    want[e] = dict(scenario=e, env=e, ordinal=0, outcome=int(info[e]), steps=int(steps[e]), subgoals=int(st["cursor"][e]),
                                   collisions=int(coll[e]), total_score=st["total_score"][e], path_len=st["path_len"][e],
                                   start2goal=float(dist(s0, g)), planner_len=plen, final_dist=float(dist(p, g)), energy=en[e])
            if len(want) == N:
                break
        assert len(want) == N and coll.sum() > 0
        rec = env.records()
        assert list(rec["slot"]) == list(range(N))
        for e in range(N):
            for k in FIELDS:
                got = rec[k][e]
                assert np.asarray(got).tobytes() == np.asarray(want[e][k], np.asarray(got).dtype).tobytes(), (e, k, got, want[e][k])
        assert env.obstacles()[2] == t + 1
    finally:
        env.close()


def compose(env, n, first, act):
    """The suite through existing calls: auto-reset with stride N, records on, act on all N rows every iteration."""
    env.set_reset_stride(env.n)
    env.set_records(n)
    env.reset(first)
    obs = env.observe()
    for it in range(100000):
        a, kind = act(obs)
        obs = env.step(a, kind=kind)["obs"]
        if it % 16 == 15 and env.records(clear=False)["slot"].size >= n:
            break
    rec = env.records(clear=False)
    assert list(rec["slot"][:n]) == list(range(n))
    return {k: rec[k][:n] for k in FIELDS}


def moving_eval_env(env_golden, env27_golden, N, P, auto_reset):
    city, params = short_episode_env(env_golden, env27_golden)
    env = engine.EnvBatch(city, params, N, max_subgoals=64, auto_reset=auto_reset)
    sc = env.make_scenarios(P, seed=5)
    env.set_pool(sc["start"], sc["goal"], sc["heading"], sc["sub"], sc["n_sub"])
    vel = np.zeros((city.buildings.shape[0], 3))
    vel[:, :2] = np.random.default_rng(12).normal(0, 4, (city.buildings.shape[0], 2))
    env.set_motion(vel, positions=city.buildings[:, :3])  # the same start before each run
    return env


@pytest.mark.parametrize("route", ["fp32", "tc", "sac_mean"])
def test_eval_under_motion_equals_composition(env_golden, env27_golden, route):
    """eval_run (fp32 and tensor-core routes) and sac_eval_run(mean_action=True) with a moving table equal the same suite driven
    through observe / act / step from the same table, bit for bit; the evaluation advances the table once per iteration."""
    N, P, n, first = 64, 300, 150, 290
    if route == "sac_mean":
        S = sac(trainers=2)
        S.init_params(4)
        E1 = moving_eval_env(env_golden, env27_golden, N, P, False)
        res = engine.sac_eval_run(E1, S, n, first_scenario=first, mean_action=True)
        act = lambda o: (S.act(o, mean=True), _lib.ACT_CONT_F32X2)  # noqa: E731
    else:
        L = learner((100, [64, 64], 27, False))
        L.init_params(3)
        if route == "fp32":
            L.set_tensor_cores(False)
            assert L.route(N)["tc_fwd"] is None
        else:
            assert L.route(N)["tc_fwd"] is not None
        E1 = moving_eval_env(env_golden, env27_golden, N, P, False)
        res = engine.eval_run(E1, L, n, first_scenario=first)
        act = lambda o: (L.act(o, 0.0, is_train=False), _lib.ACT_DISCRETE27)  # noqa: E731
    assert res["unfinished"] == 0 and res["n_records"] == n
    assert E1.obstacles()[2] == res["iterations"] > MAX_STEP
    E2 = moving_eval_env(env_golden, env27_golden, N, P, True)
    want = compose(E2, n, first, act)
    for k in FIELDS:
        assert_same(res["records"][k], want[k], "%s: %s" % (route, k))
    assert (res["records"]["collisions"] > 0).any()
    E1.close(); E2.close()
