"""The CUDA sources' include graph keeps the SAC learner and the shared optimiser apart from the Q-network learner: neither
sac.cu nor what it includes reaches learner.cuh (the Q-network's handle, tensor-core net and Q-head arithmetic), so a change
there cannot recompile or break SAC; and the optimiser / exchange header does not reach the SAC learner either."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dqn-based-uav-3d_path_planer_b200", "csrc")
INCLUDE = re.compile(r'^\s*#\s*include\s+"([^"]+)"', re.M)


def closure(name):
    """Every file under csrc/ that `name` includes, directly or through another file, `name` itself excluded."""
    seen, todo = set(), [os.path.normpath(os.path.join(CSRC, name))]
    while todo:
        path = todo.pop()
        with open(path) as f:
            for inc in INCLUDE.findall(f.read()):
                dep = os.path.normpath(os.path.join(os.path.dirname(path), inc))
                if dep not in seen and os.path.dirname(dep) == os.path.normpath(CSRC):
                    seen.add(dep)
                    todo.append(dep)
    return {os.path.basename(p) for p in seen}


@pytest.mark.parametrize("name", ["sac.cu", "sac.cuh", "mlp_tile.cuh", "net.cuh", "optim.cuh", "optim.cu"])
def test_shared_and_sac_sources_do_not_reach_the_q_learner(name):
    assert os.path.exists(os.path.join(CSRC, name)), name
    assert "learner.cuh" not in closure(name)


def test_optimiser_header_does_not_reach_sac():
    assert "sac.cuh" not in closure("optim.cuh")


def test_closure_follows_includes_transitively():
    """The walk itself: train.cu reaches learner.cuh directly and net.cuh only through learner.cuh or sac.cuh."""
    reach = closure("train.cu")
    assert {"learner.cuh", "sac.cuh", "net.cuh", "optim.cuh", "common.cuh"} <= reach
    assert "train.cu" not in reach
