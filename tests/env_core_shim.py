"""csrc/env_core.cuh (the source the CUDA env kernel instantiates per env) compiled for the host by tests/host_shim: the
module fixture `shim` builds and loads it, shim_step steps an OracleBatch through it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle as O
from conftest import ROOT

SHIM_DIR = os.path.join(ROOT, "tests", "host_shim")
SHIM_SO = os.path.join(SHIM_DIR, "_build", "libenv_core_host.so")


@pytest.fixture(scope="module")
def shim():
    os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(SHIM_DIR, "env_core_host.cpp"), "-o", SHIM_SO])
    return C.CDLL(SHIM_SO)


def shim_step(shim, city, params, b, actions, mode, want_obs=True):
    n = b.n
    rew = np.zeros(n); done = np.zeros(n, np.uint8); info = np.zeros(n, np.uint8); coll = np.zeros(n, np.uint8)
    obs = np.zeros((n, 100), np.float32)
    st = b._struct()
    acts = None if actions is None else np.ascontiguousarray(actions, np.float64)
    shim.shim_step(C.c_double(city.c.width), C.c_double(city.c.h), C.c_int(city.buildings.shape[0]),
                   O._p(city.buildings, C.c_double), C.c_double(params.max_v), C.c_double(params.min_v),
                   C.c_double(params.steering), C.c_double(params.climb_rate), C.c_int(params.max_step),
                   C.c_int(mode), C.byref(st), O._p(acts, C.c_double) if acts is not None else None,
                   O._p(rew, C.c_double), O._p(done, C.c_uint8), O._p(info, C.c_uint8), O._p(coll, C.c_uint8),
                   O._p(obs, C.c_float) if want_obs else None)
    return rew, done, info, coll, obs
