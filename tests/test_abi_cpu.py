"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads, exports every symbol
include/uavrl.h declares, and refuses to run without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import uavrl_b200
from uavrl_b200 import _lib, engine
from conftest import ROOT


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "uavrl.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(uavrl_[a-z_0-9]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(L, s), "include/uavrl.h declares %s but the library does not export it" % s
        assert s in _lib.SIGNATURES, "%s has no ctypes signature in _lib.py" % s
    assert b"sm_90a" in L.uavrl_version()


def test_sass_is_sm_90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    city = engine.City(500, 500, 100, np.zeros((1, 5)))
    with pytest.raises(uavrl_b200.UavrlError, match="no CUDA device"):
        engine.EnvBatch(city, engine.UavParams(), 4)
    cfg = _lib.LearnerConfig()
    cfg.in_dim, cfg.n_hidden, cfg.n_actions, cfg.batch_size, cfg.replay_capacity = 100, 1, 27, 64, 1000
    cfg.hidden[0] = 64
    h = C.c_void_p()
    assert _lib.lib().uavrl_learner_create(C.byref(cfg), C.byref(h)) == -2


def test_argument_validation_without_gpu():
    L = _lib.lib()
    assert L.uavrl_env_create(None, None) == -1
    assert b"null" in L.uavrl_last_error()
    cfg = _lib.EnvConfig()
    cfg.n_envs, cfg.max_subgoals, cfg.n_buildings = 4, 8, 100     # > 64 cylinders is rejected up front
    h = C.c_void_p()
    assert L.uavrl_env_create(C.byref(cfg), C.byref(h)) == -1
    # the two removed scheduling variants keep their setters for ABI compatibility: 0 is accepted, anything else refused
    for setter in (L.uavrl_set_fuse_act_env, L.uavrl_set_fuse_dw_adam):
        assert setter(0) == 0
        assert setter(1) == -1 and b"removed" in L.uavrl_last_error()


def test_host_scenario_generator(env_golden):
    """uavrl_make_scenarios is host code (RRT): runs without a GPU; check reference invariants."""
    g = env_golden
    cfg = _lib.EnvConfig()
    b = np.ascontiguousarray(g["buildings"])
    cfg.n_envs, cfg.max_subgoals = 1, 64
    cfg.len, cfg.width, cfg.h = g["dims"]
    cfg.max_v, cfg.min_v, cfg.steering_angle, cfg.max_step = g["uav_params"][0], g["uav_params"][1], g["uav_params"][2], 150
    cfg.n_buildings, cfg.buildings_host = b.shape[0], b.ctypes.data_as(C.POINTER(C.c_double))
    P, K = 64, 64
    start = np.zeros((P, 3)); goal = np.zeros((P, 3)); heading = np.zeros(P); sub = np.zeros((P, K, 3))
    n_sub = np.zeros(P, np.int32)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    rc = _lib.lib().uavrl_make_scenarios(C.byref(cfg), 7, P, 30, vp(start), vp(goal), vp(heading), vp(sub), vp(n_sub))
    assert rc == 0, _lib.lib().uavrl_last_error()
    import oracle as O
    city = O.OracleCity(g["dims"][0], g["dims"][1], g["dims"][2], b)
    assert (start[:, 0] >= 10).all() and (start[:, 0] <= 210).all() and (start[:, 1] >= 1).all() and (start[:, 1] <= 10).all()
    assert (goal[:, 0] >= 330).all() and (goal[:, 0] <= 490).all() and (goal[:, 1] >= 420).all() and (goal[:, 1] <= 490).all()
    assert (heading >= 0).all() and (heading < 2 * np.pi).all()
    for s in range(P):
        k = n_sub[s]
        assert 2 <= k <= K
        assert np.array_equal(sub[s, 0], start[s]) and np.array_equal(sub[s, k - 1], goal[s])   # RRT.py:98-103
        seg = np.linalg.norm(np.diff(sub[s, :k], axis=0), axis=1)
        assert (seg <= 30 + 1e-9).all()                                                          # steer(), step 30
        assert city.threaten_rate(sub[s, :k]).sum() == 0                                         # nodes are collision free
    assert 8 <= np.median(n_sub) <= 40


def test_scenario_generator_matches_reference_statistics(env_golden):
    """Statistical pin of rrt_core.cuh against 400 resets of the reference's own UAV.reset -> RRT
    (tests/golden/rrt_golden.npz): sub-goal counts, chain length and detour ratio follow the same distributions
    (two-sample Kolmogorov-Smirnov), segment lengths never exceed the RRT step."""
    from scipy import stats
    g = env_golden
    ref = np.load(os.path.join(ROOT, "tests", "golden", "rrt_golden.npz"))
    cfg = _lib.EnvConfig()
    b = np.ascontiguousarray(g["buildings"])
    cfg.n_envs, cfg.max_subgoals = 1, 64
    cfg.len, cfg.width, cfg.h = g["dims"]
    cfg.max_v, cfg.min_v, cfg.steering_angle, cfg.max_step = g["uav_params"][0], g["uav_params"][1], g["uav_params"][2], 150
    cfg.n_buildings, cfg.buildings_host = b.shape[0], b.ctypes.data_as(C.POINTER(C.c_double))
    P, K = 2000, 64
    start = np.zeros((P, 3)); goal = np.zeros((P, 3)); heading = np.zeros(P); sub = np.zeros((P, K, 3))
    n_sub = np.zeros(P, np.int32)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    assert _lib.lib().uavrl_make_scenarios(C.byref(cfg), 99, P, 30, vp(start), vp(goal), vp(heading), vp(sub), vp(n_sub)) == 0
    chain = np.zeros(P); seg_max = np.zeros(P)
    for s in range(P):
        seg = np.linalg.norm(np.diff(sub[s, :n_sub[s]], axis=0), axis=1)
        chain[s], seg_max[s] = seg.sum(), seg.max()
    straight = np.linalg.norm(goal - start, axis=1)
    assert seg_max.max() <= 30 + 1e-9 and ref["seg_max"].max() <= 30 + 1e-9
    for ours, theirs, what in ((n_sub, ref["n_sub"], "n_sub"), (chain, ref["chain"], "chain length"),
                               (chain / straight, ref["chain"] / ref["straight"], "detour ratio"),
                               (start[:, 0], ref["start"][:, 0], "start x"), (goal[:, 1], ref["goal"][:, 1], "goal y")):
        p = stats.ks_2samp(ours, theirs).pvalue
        assert p > 1e-3, "%s: KS p=%.2e (ours mean %.3f, reference mean %.3f)" % (what, p, np.mean(ours), np.mean(theirs))
