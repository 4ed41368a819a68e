"""The CUDA sources' include graph keeps the SAC learner, the shared optimiser and the replay store with its prioritised-replay
trees apart from the Q-network learner: none of them reaches learner.cuh (the Q-network's handle, tensor-core net and Q-head
arithmetic), so a change there cannot recompile or break them; and neither the optimiser / exchange header nor the replay and
tree headers reach the SAC learner."""
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


@pytest.mark.parametrize("name", ["sac.cu", "sac.cuh", "mlp_tile.cuh", "net.cuh", "optim.cuh", "optim.cu",
                                  "per.cu", "per.cuh", "replay.cu", "replay.cuh"])
def test_shared_and_sac_sources_do_not_reach_the_q_learner(name):
    assert os.path.exists(os.path.join(CSRC, name)), name
    assert "learner.cuh" not in closure(name)


def test_optimiser_header_does_not_reach_sac():
    assert "sac.cuh" not in closure("optim.cuh")


@pytest.mark.parametrize("name", ["per.cuh", "replay.cuh"])
def test_replay_headers_do_not_reach_sac(name):
    assert os.path.exists(os.path.join(CSRC, name)), name
    assert "sac.cuh" not in closure(name)


def test_closure_follows_includes_transitively():
    """The walk itself: train.cu reaches learner.cuh directly and net.cuh only through learner.cuh or sac.cuh."""
    reach = closure("train.cu")
    assert {"learner.cuh", "sac.cuh", "net.cuh", "optim.cuh", "common.cuh"} <= reach
    assert "train.cu" not in reach
