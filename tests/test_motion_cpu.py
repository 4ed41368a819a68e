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


def test_host_compiled_obstacle_run_matches_golden(g, tmp_path):
    """env_core.cuh's obstacle_run (the code the kernel runs) compiled for the host, run from each episode's first table,
    reproduces every table the reference recorded, bit for bit."""
    so = str(tmp_path / "libmotion_host.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", SHIM_SRC, "-o", so])
    lib = C.CDLL(so)
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
