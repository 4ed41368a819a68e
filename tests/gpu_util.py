"""Shared helpers for the -m gpu parity tests (CUDA path vs the CPU oracle / golden vectors)."""
import contextlib
import importlib
import os

import numpy as np
import torch

import oracle as O
import uavrl_b200  # noqa: F401
from uavrl_b200 import engine


def city_and_params(env_golden, env27_golden):
    g = env_golden
    city = engine.City(g["dims"][0], g["dims"][1], g["dims"][2], g["buildings"])
    p = g["uav_params"]
    params = engine.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    ocity = O.OracleCity(g["dims"][0], g["dims"][1], g["dims"][2], g["buildings"])
    oparams = O.UavParams(p[0], p[1], p[2], float(env27_golden["climb_rate"]), int(p[3]))
    return city, params, ocity, oparams


def assert_close64(a, b, tol=1e-9, what=""):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    err = np.abs(a - b) / np.maximum(1.0, np.abs(b))
    assert err.max() <= tol, (what, float(err.max()), int(err.argmax()))


BIN = np.r_[11:86, 90:95]          # the 80 occupancy probes: exact {0,1}
REAL = np.r_[0:11, 86:90, 95:100]  # real-valued entries


def assert_obs(got, want64, what=""):
    """got: fp32 obs from the GPU; want64: fp64 obs of the oracle/reference.  North-star tolerance:
    1e-5 on real-valued entries, occupancy bits exact."""
    got = np.asarray(got); want64 = np.asarray(want64, np.float64)
    assert np.array_equal(got[..., BIN], want64[..., BIN].astype(np.float32)), what
    np.testing.assert_allclose(got[..., REAL], want64[..., REAL], rtol=1e-5, atol=1e-5, err_msg=what)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def env_plugin(model_path):
    """The env plug-in module, run from the repository root, whose trainers read a small batch and replay, no periodic
    save and checkpoints under model_path."""
    cwd = os.getcwd()
    os.chdir(ROOT)
    mod = importlib.import_module("uavrl_b200.plugins.PathPlan_City_B200")
    orig = mod.XML2Dict

    def patched(path):
        d = orig(path)
        if "Trainer" in d and isinstance(d["Trainer"], dict):
            d["Trainer"].update(Batch_Size="16", replay_size="512", save_loop="0", model_path=str(model_path))
        return d
    mod.XML2Dict = patched
    try:
        yield mod
    finally:
        mod.XML2Dict = orig
        os.chdir(cwd)
