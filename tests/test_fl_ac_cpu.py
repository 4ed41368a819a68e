"""Federated_Learning_AC (Envs/PathPlan_City.py:590-601) restated in numpy and pinned, bit for bit, to the reference's own run
(tests/golden/fl_ac_golden.npz, made by make_fl_ac_golden.py on real reference SAC trainers).  No GPU: this fixes what the
device kernel (uavrl_sac_federate_actors) must compute before any GPU test compares against it."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fl_ac_golden.npz")


def federate_actors(actors):
    """Every actor <- the float32 sum theta_0 + theta_1 + ... + theta_{G-1}, added left to right in trainer order.  The
    reference's division by G assigns into a temporary state_dict and is lost, so nothing is divided."""
    actors = np.asarray(actors, np.float32)
    s = actors[0].copy()
    for g in range(1, actors.shape[0]):
        s = np.add(s, actors[g], dtype=np.float32)
    return np.broadcast_to(s, actors.shape).copy()


def test_restatement_matches_reference_golden():
    g = np.load(GOLDEN)
    G = int(g["G"])
    assert g["actor0"].shape == g["actor1"].shape == (G, 64 * 100 + 64 + 2 * (2 * 64 + 2))
    out = federate_actors(g["actor0"])
    assert np.array_equal(out.view(np.uint32), g["actor1"].view(np.uint32))


def test_golden_is_the_sum_not_the_mean():
    g = np.load(GOLDEN)
    G = int(g["G"])
    mean = (federate_actors(g["actor0"])[0] / np.float32(G)).astype(np.float32)
    assert not np.array_equal(g["actor1"][0], mean)
    assert all(np.array_equal(row, g["actor1"][0]) for row in g["actor1"])


def test_restatement_adds_left_to_right():
    """With full float32 mantissas the summation order shows: the restatement is the in-order sum, not a pairwise one."""
    rng = np.random.default_rng(0)
    a = rng.normal(0, 1, (7, 4096)).astype(np.float32)
    out = federate_actors(a)[0]
    seq = a[0]
    for x in a[1:]:
        seq = (seq + x).astype(np.float32)
    assert np.array_equal(out, seq)
    pairwise = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + a[6])
    assert not np.array_equal(out, pairwise.astype(np.float32))
    assert np.array_equal(federate_actors(a[:1]), a[:1])           # one trainer keeps its actor
