"""The numpy restatement of the selective federated aggregation (tests/fl_restatement.py) against the reference's own
run (fl_golden.npz, Envs/PathPlan_City.py:644-684).  The GPU federation tests judge the device with this restatement,
so it is pinned here first: the same selections, bit-identical parameters after, and round order that matters."""
import os

import numpy as np
import pytest

import fl_restatement as flr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fl_golden.npz")


@pytest.fixture(scope="module")
def fl_golden():
    return np.load(GOLDEN)


def case(g, name):
    k = lambda s: g["%s_%s" % (name, s)]                  # noqa: E731
    return dict(local0=k("local0"), local1=k("local1"), probes=k("probes"), chosen=k("chosen"),
                hidden=[int(h) for h in k("hidden")], dueling=bool(k("dueling")))


@pytest.mark.parametrize("name", ["ddqn5", "duel6"])
def test_restatement_matches_reference(fl_golden, name):
    c = case(fl_golden, name)
    theta, chosen, M = flr.federate(c["local0"], c["probes"], 100, c["hidden"], 27, c["dueling"])
    assert np.array_equal(chosen, c["chosen"])
    assert np.array_equal(theta, c["local1"])
    assert (np.diag(M) == 0).all()


@pytest.mark.parametrize("name", ["ddqn5", "duel6"])
def test_round_order_discriminates(fl_golden, name):
    c = case(fl_golden, name)
    jac, _, _ = flr.federate(c["local0"], c["probes"], 100, c["hidden"], 27, c["dueling"], jacobi=True)
    assert not np.array_equal(jac, c["local1"])


def test_exact_tie_keeps_lower_index(fl_golden):
    c = case(fl_golden, "duel6")
    assert np.array_equal(c["local0"][4], c["local0"][5])
    assert c["chosen"][0].tolist() == [1, 4]
    _, _, M = flr.federate(c["local0"], c["probes"], 100, c["hidden"], 27, c["dueling"])
    assert M[0, 4] == M[0, 5]


def test_average_is_in_order_float32(fl_golden):
    """The average is a left-to-right float32 sum and one division, not a pairwise sum or a product with 1 / (k + 1)."""
    c = case(fl_golden, "ddqn5")
    th = c["local0"].astype(np.float32)
    a = flr.average(th, 0, [3, 1])
    assert np.array_equal(a, ((th[0] + th[3]) + th[1]) / np.float32(3))
    k1 = ((th[0] + th[3]) + th[1]) * np.float32(1.0 / 3.0)
    assert not np.array_equal(a, k1)


def test_small_groups_are_unchanged(fl_golden):
    c = case(fl_golden, "ddqn5")
    for G in (1, 2):
        theta, chosen, _ = flr.federate(c["local0"][:G], c["probes"][:G], 100, c["hidden"], 27, False)
        assert np.array_equal(theta, c["local0"][:G]) and (chosen == -1).all()
