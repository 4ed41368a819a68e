"""CPU check of the built library's SASS: in the headline tensor-core kernels (act pass, DQN / double-DQN / dueling
training chain with fused TD target) every layer product is ONE unbroken wgmma chain -- 3 x k-steps HGMMA behind one
WARPGROUP.ARRIVE, closed by one gsb0 wait -- and not a chain that ptxas cut into groups of a few instructions.  In the
generic (runtime-K) instances ptxas has not serialised the wgmma (C7515: a wait behind every HGMMA)."""
import os
import re
import shutil
import subprocess

import pytest

from uavrl_b200 import _lib

# (ACT, DUELING, FIXED) / (NPRE, DUELING, FIXED): the variants the shipped networks run
KERNELS = [
    "_ZN5uavrl19tc_forward_kernel_tILb1ELb0ELb1EEEvNS_5TcNetENS_6TcArgsE",
    "_ZN5uavrl19tc_forward_kernel_tILb1ELb1ELb1EEEvNS_5TcNetENS_6TcArgsE",
    "_ZN5uavrl15tc_train_kernelILi1ELb0ELb1EEEvNS_5TcNetENS_11TcTrainArgsE",
    "_ZN5uavrl15tc_train_kernelILi2ELb0ELb1EEEvNS_5TcNetENS_11TcTrainArgsE",
    "_ZN5uavrl15tc_train_kernelILi2ELb1ELb1EEEvNS_5TcNetENS_11TcTrainArgsE",
]
KSTEPS = (4, 8, 13, 16)          # wgmma.cuh mma_fixed
# the generic (FIXED = false) instances of every tensor-core kernel
GENERIC = (["_ZN5uavrl19tc_forward_kernel_tILb%dELb%dELb0EEEvNS_5TcNetENS_6TcArgsE" % (a, d) for a in (0, 1) for d in (0, 1)]
           + ["_ZN5uavrl16tc_loss_kernel_tILb%dELb0EEEvNS_5TcNetENS_6TcArgsE" % d for d in (0, 1)]
           + ["_ZN5uavrl15tc_train_kernelILi%dELb%dELb0EEEvNS_5TcNetENS_11TcTrainArgsE" % (n, d) for n in (0, 1, 2) for d in (0, 1)])


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    pytest.skip("cuobjdump not found")


@pytest.mark.parametrize("kernel", KERNELS)
def test_layer_products_are_unbroken_chains(kernel):
    sass = subprocess.run([_cuobjdump(), "-sass", "-fun", kernel, _lib.LIB_PATH], capture_output=True, text=True).stdout
    ops = re.findall(r"\b(WARPGROUP\.ARRIVE|HGMMA[^;]*)", sass)
    assert ops, "no SASS for " + kernel
    groups, cur = [], None
    for op in ops:
        if op.startswith("WARPGROUP"):
            assert cur is None, "WARPGROUP.ARRIVE inside an open wgmma group"
            cur = 0
        else:
            assert cur is not None, "HGMMA outside a group"
            cur += 1
            if "gsb0" in op:
                groups.append(cur)
                cur = None
    assert cur is None
    assert groups and all(g in [3 * k for k in KSTEPS] for g in groups), groups


@pytest.mark.parametrize("kernel", GENERIC)
def test_generic_products_are_not_serialised(kernel):
    # Serialised (ptxas C7515), every HGMMA is its own group with its own WARPGROUP.DEPBAR.  The runtime-K chains wait a few
    # times per kernel (3 DEPBAR for 66 HGMMA in the act kernel of a 2-hidden-layer network).
    sass = subprocess.run([_cuobjdump(), "-sass", "-fun", kernel, _lib.LIB_PATH], capture_output=True, text=True).stdout
    hgmma = re.findall(r"\bHGMMA", sass)
    depbar = re.findall(r"WARPGROUP\.DEPBAR", sass)
    assert hgmma, "no SASS for " + kernel
    assert len(depbar) * 4 < len(hgmma), (len(hgmma), len(depbar))
