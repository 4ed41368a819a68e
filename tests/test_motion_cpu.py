"""Moving obstacles without a GPU: the oracle's table and step order against the reference (tests/golden/motion_golden.npz,
tests/golden/make_motion_golden.py), env_core.cuh's obstacle_run compiled for the host, and the plug-in's XML surface."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import motion_oracle as MO
import oracle as O
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "motion_golden.npz")
SHIM_SRC = os.path.join(ROOT, "tests", "host_shim", "motion_host.cpp")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def episodes(g, c):
    i = 0
    while "cfg%d_ep%d_action" % (c, i) in g:
        pre = "cfg%d_ep%d_" % (c, i)
        yield {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
        i += 1


@pytest.mark.parametrize("c", [0, 1, 2], ids=["continuous", "apf", "discrete27"])
def test_oracle_reproduces_reference_loop(g, c):
    """The oracle with the table set to the reference's after its first run(): per step the reward, masks, position, sub-goal
    queue and table bit for bit, its observation equal to the reference's state_test of the next iteration, and the
    reference's Move_Agent next_state (taken before the next run()) equal to the observation on the old table -- which
    differs from state_test at some steps: the port's documented deviation."""
    dims, p = g["dims"], g["uav_params"]
    params = O.UavParams(p[0], p[1], p[2], float(g["climb_rate"]), int(p[3]))
    mode = O.ACT_DISCRETE27 if c == 2 else O.ACT_CONTINUOUS
    total, deviating = 0, 0
    for ep in episodes(g, c):
        K = len(ep["action"])
        mc = MO.MovingCity(dims[0], dims[1], dims[2], g["buildings"], ep["tab1"], g["obstacle_v"][:, 2], apf=(c == 1))
        try:
            b = O.OracleBatch(mc.city, params, 1, ep["sub"].shape[0])
            b.reset(ep["start"][None], ep["goal"][None], [ep["heading"]], ep["sub"][None], [ep["n_sub"]], [ep["alias0"]])
            assert np.array_equal(b.state(want64=True)[1][0], ep["state_test"][0])
            for t in range(K):
                assert MO.table_digest(mc.tab) == ep["tab_digest"][t].tobytes(), (c, t)
                rew, done, info, coll, _ = b.step_([ep["action"][t]], mode, want_obs=False)
                assert rew[0] == ep["reward"][t], (c, t, rew[0], ep["reward"][t])
                assert (done[0], info[0], coll[0]) == (ep["done_ret"][t], ep["info"][t], ep["collision"][t]), (c, t)
                assert (b.px[0], b.py[0], b.pz[0]) == (ep["px"][t], ep["py"][t], ep["pz"][t]), (c, t)
                if "subq" in ep:
                    nleft = int(b.n_sub[0] - b.cursor[0])
                    assert np.array_equal(b.sub[0, b.cursor[0]:b.n_sub[0]], ep["subq"][t][:nleft]), (c, t)
                old = b.state(want64=True)[1][0]
                assert np.array_equal(old, ep["next_state"][t]), (c, t)
                mc.advance()
                if t + 1 < K:
                    new = b.state(want64=True)[1][0]
                    assert np.array_equal(new, ep["state_test"][t + 1]), (c, t)
                    deviating += int(not np.array_equal(ep["next_state"][t], ep["state_test"][t + 1]))
                total += 1
        finally:
            mc.close()
    assert total > 400 and deviating > 0, (total, deviating)


def test_golden_reflects_on_every_wall(g):
    """A reflection at x = 0 turns vx from negative to positive, at x = len the other way (likewise y): the golden's velocity
    sign bits before and after each run() show all four."""
    walls = set()
    for c in range(int(g["n_cfg"])):
        for ep in episodes(g, c):
            after = ep["vsign"].astype(np.int32)
            before = np.concatenate([MO.velocity_signs(ep["tab0"])[None].astype(np.int32), after[:-1]])
            moving = (ep["tab0"][:, 2:] != 0)
            for bit, axis, (lo, hi) in ((1, 0, ("x0", "xlen")), (2, 1, ("y0", "ywidth"))):
                b_neg, a_neg = (before & bit) != 0, (after & bit) != 0
                if (b_neg & ~a_neg & moving[:, axis]).any(): walls.add(lo)
                if (~b_neg & a_neg & moving[:, axis]).any(): walls.add(hi)
    assert walls == {"x0", "xlen", "y0", "ywidth"}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """env_core.cuh's obstacle_run (the code the kernel runs) compiled for the host."""
    so = str(tmp_path_factory.mktemp("motion_host") / "libmotion_host.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", SHIM_SRC, "-o", so])
    return C.CDLL(so)


def test_host_compiled_obstacle_run_matches_golden(g, shim):
    """obstacle_run compiled for the host, run from each episode's first table, reproduces every table the reference
    recorded, bit for bit."""
    lib = shim
    dims = g["dims"]
    n = 0
    for c in range(int(g["n_cfg"])):
        for ep in episodes(g, c):
            rows = np.ascontiguousarray(ep["tab0"], np.float64).copy()
            for t in range(len(ep["tab_digest"])):
                lib.shim_obstacle_run(C.c_int(rows.shape[0]), rows.ctypes.data_as(C.c_void_p), C.c_double(dims[0]),
                                      C.c_double(dims[1]), C.c_int(1))
                assert MO.table_digest(rows) == ep["tab_digest"][t].tobytes(), (c, t)
                n += 1
    assert n > 1000


def edge_rows(L, W, rng):
    """Hand rows (x, y, vx, vy) of an L x W box: centres on every wall and corner, |v| exactly L / W (wall to wall every run),
    x + vx landing exactly on 0 or L (not a reflection), signed zeros and subnormal velocities."""
    tiny = np.nextafter(0.0, 1.0)
    rows = []
    for x, y in ((0.0, W / 3), (L, W / 3), (L / 3, 0.0), (L / 3, W), (0.0, 0.0), (L, 0.0), (0.0, W), (L, W), (-0.0, -0.0)):
        rows += [(x, y, rng.uniform(-L, L), rng.uniform(-W, W)), (x, y, L, W), (x, y, -L, -W), (x, y, L, -W), (x, y, -0.0, 0.0)]
    rows += [(L / 2, W / 2, L, W), (L / 4, 3 * W / 4, -L, W)]
    for x in (L / 4, L / 2, 0.375 * L):                     # dyadic fractions: x - x and x + (L - x) are exact
        rows += [(x, W / 2, -x, 0.0), (x, W / 2, L - x, 0.0)]
    for y in (W / 4, 0.625 * W):
        rows += [(L / 2, y, 0.0, -y), (L / 2, y, 0.0, W - y)]
    rows += [(0.0, 0.0, -tiny, -tiny), (L, W, tiny, tiny), (0.0, W, tiny, -tiny), (L / 2, W / 2, -0.0, -0.0),
             (0.0, 0.0, 0.0, -0.0), (L, W / 2, -tiny, 0.0)]
    return np.array(rows, np.float64)


@pytest.mark.parametrize("L,W", [(300.0, 800.0), (800.0, 300.0), (1.0, 1000.0), (500.0, 500.0)])
def test_host_compiled_obstacle_run_on_non_square_boxes(shim, L, W):
    """obstacle_run compiled for the host against motion_oracle.obstacle_run, bit for bit after every run, on random tables
    (|vx| <= len, |vy| <= width) and the hand edge rows; after every run the centres lie in [0, len] x [0, width] and each
    velocity component keeps its magnitude (only its sign may flip); over the runs every wall reflects some row.  A len /
    width swap anywhere in the rule fails the first three boxes."""
    rng = np.random.default_rng(int(L * 7 + W))
    n = 96
    rnd = np.zeros((n, 4))
    rnd[:, 0] = rng.uniform(0, L, n); rnd[:, 1] = rng.uniform(0, W, n)
    rnd[:, 2] = rng.uniform(-L, L, n) * rng.choice([1.0, 0.1, 0.01], n)
    rnd[:, 3] = rng.uniform(-W, W, n) * rng.choice([1.0, 0.1, 0.01], n)
    edge = edge_rows(L, W, rng)
    tab = np.concatenate([rnd, edge])
    dev = np.ascontiguousarray(tab.copy())
    mag = np.abs(tab[:, 2:]).copy()
    walls = dict.fromkeys(("x0", "xlen", "y0", "ywidth"), 0)
    runs = 0
    for t in range(80):
        before = tab.copy()
        MO.obstacle_run(tab, L, W)
        shim.shim_obstacle_run(C.c_int(dev.shape[0]), dev.ctypes.data_as(C.c_void_p), C.c_double(L), C.c_double(W), C.c_int(1))
        assert MO.table_digest(dev) == MO.table_digest(tab), (L, W, t, np.nonzero((dev != tab).any(1))[0])
        assert ((tab[:, 0] >= 0) & (tab[:, 0] <= L) & (tab[:, 1] >= 0) & (tab[:, 1] <= W)).all(), (L, W, t)
        assert np.array_equal(np.abs(tab[:, 2:]), mag), (L, W, t)
        for k, v in MO.wall_reflections(before, tab).items():
            walls[k] += v
        runs += tab.shape[0]
    assert runs >= 10000 and min(walls.values()) > 0, walls
    # landing exactly on a wall is not a reflection: the first run keeps those velocities
    one = edge.copy()
    MO.obstacle_run(one, L, W)
    land = (edge[:, 3] == 0.0) & (edge[:, 1] == W / 2) & ((edge[:, 0] + edge[:, 2] == 0.0) | (edge[:, 0] + edge[:, 2] == L))
    assert land.sum() >= 4 and np.array_equal(one[land, 2], edge[land, 2]) and np.isin(one[land, 0], (0.0, L)).all()


def test_probe_points_are_the_observation_probes():
    """motion_oracle.probe_points in slot order: the oracle's threaten_rate on them equals the occupancy bits of the oracle's
    own observation, on a dense city with UAVs next to cylinders and the box edges."""
    rng = np.random.default_rng(2)
    L, W, H = 300.0, 800.0, 80.0
    b = np.zeros((40, 5))
    b[:, 0] = rng.uniform(0, W, 40); b[:, 1] = rng.uniform(0, W, 40)
    b[:, 2] = 1.0; b[:, 3] = rng.uniform(4, 20, 40); b[:, 4] = rng.uniform(3, 60, 40)
    city = O.OracleCity(L, W, H, b)
    n = 64
    ob = O.OracleBatch(city, O.UavParams(), n, 2)
    start = np.stack([rng.uniform(-5, W + 5, n), rng.uniform(-5, W + 5, n), rng.uniform(0, 12, n)], 1)
    start[:8, 0] = [0.0, 19.5, 20.0, W - 20.0, W, 10.0, 5.0, 1.0]
    ob.reset(start, start + 50, rng.uniform(0, 6, n), np.repeat(start[:, None], 2, 1), np.full(n, 2))
    obs = ob.state(want64=True)[1]
    pts = MO.probe_points(ob.px, ob.py, ob.pz)
    bits = city.threaten_rate(pts.reshape(-1, 3)).reshape(n, 80)
    assert np.array_equal(bits, obs[:, MO.PROBE_SLOT].astype(np.uint8))
    assert 0 < bits.sum() < bits.size


def write_xml_variants(tmp_path):
    """The shipped buildings XML with a <v> on two obstacles, and the shipped UAV XML with APF_Enabled = 1."""
    cfg = os.path.join(ROOT, "configs")
    txt = open(os.path.join(cfg, "buildings.xml")).read()
    parts = txt.split("</Threaten>")
    parts[0] += "<v><x>1.5</x><y>-0.25</y><z>0.5</z></v>"
    parts[2] += "<v><x>-2</x></v>"
    bv = tmp_path / "buildings_v.xml"
    bv.write_text("</Threaten>".join(parts))
    uav = tmp_path / "UAV_apf.xml"
    uav.write_text(open(os.path.join(cfg, "UAV_B200.xml")).read().replace("<APF_Enabled>0</APF_Enabled>", "<APF_Enabled>1</APF_Enabled>"))
    return str(bv), str(uav)


def test_plugin_reads_obstacle_velocities_and_refuses_apf_without_them(tmp_path):
    from uavrl_b200.plugins import xmlconfig
    from uavrl_b200.plugins.PathPlan_City_B200 import PathPlan_City_B200, buildings_from_dict, obstacle_v_from_dict
    bv, uav = write_xml_variants(tmp_path)
    shipped = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", "buildings.xml"))["buildings"]
    v, has = obstacle_v_from_dict(shipped)
    assert not has and not v.any() and v.shape == (buildings_from_dict(shipped).shape[0], 3)
    v, has = obstacle_v_from_dict(xmlconfig.XML2Dict(bv)["buildings"])
    assert has and v[0].tolist() == [1.5, -0.25, 0.5] and v[2].tolist() == [-2.0, 0.0, 0.0] and not v[1].any() and not v[3:].any()
    assert np.array_equal(buildings_from_dict(xmlconfig.XML2Dict(bv)["buildings"]), buildings_from_dict(shipped))
    ed = xmlconfig.XML2Dict(os.path.join(ROOT, "configs", "PathPlan_City_B200.xml"))["simulator"]["env"]
    ed["Obstacles"]["buildings"] = os.path.join(ROOT, "configs", "buildings.xml")
    ed["Agent"]["xml_path_agent"] = uav
    ed["Agent"]["Trainer"]["Trainer_path"] = os.path.join(ROOT, "configs", "Trainer_DDQN_B200.xml")
    with pytest.raises(ValueError, match="APF_Enabled = 1 needs obstacle velocities"):
        PathPlan_City_B200(ed)
