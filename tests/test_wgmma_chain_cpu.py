"""CPU check of the built library's SASS: in the headline tensor-core kernels (act pass, DQN / double-DQN / dueling
training chain with fused TD target) every layer product is ONE unbroken wgmma chain -- 3 x k-steps HGMMA behind one
WARPGROUP.ARRIVE, closed by one gsb0 wait -- and not a chain that ptxas cut into groups of a few instructions."""
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
