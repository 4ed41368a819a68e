"""The discrete SAC update regimes (sac_discrete_restatement.regime_rows) on the CPU: every row's float64 update is finite
and has a batch clear of the ReLU kinks, and every named deviation of the update (MUTANTS) falls outside compare_step's
bounds on at least one row -- while the two +1e-8 deviations pass every row of the shape sweep, which starts from
init_state.  No GPU."""
import numpy as np
import pytest

from sac_discrete_restatement import (HP, MUTANTS, WIDEST, categorical_pick, clean_batch, compare_step, fc3, init_state, regime_batch,
                                      regime_rows, regime_seed, regime_state, sacd_update64)

ROWS = regime_rows(WIDEST[31, 128])


def regime_step(rid, shape, sk, bk, hp):
    A, hid, obs, B = shape
    rng = np.random.default_rng(regime_seed(rid))
    st = regime_state(rng, obs, hid, A, hp=hp, **sk)
    batch = regime_batch(rng, st, B, obs, hid, A, **bk)
    return st, batch


def caught(st, batch, shape, hp, mutant):
    """compare_step's complaint (what, entry, ...) about a learner computing `mutant`, or None"""
    A, hid, obs, _ = shape
    new, out = sacd_update64(st, *batch, obs, hid, A, hp)
    mnew, mout = sacd_update64(st, *batch, obs, hid, A, hp, **{mutant: True})
    try:
        compare_step(mout["losses"], mout["grads"], mnew, new, out, mutant, hp)
    except AssertionError as e:
        return e.args[0]
    return None


@pytest.mark.parametrize("rid,shape,sk,bk,hp", [r for r in ROWS if r[1][3] <= 64], ids=[r[0] for r in ROWS if r[1][3] <= 64])
def test_regime_update_finite_and_self_consistent(rid, shape, sk, bk, hp):
    """The float64 update from the regime's state is finite, and compare_step accepts it against itself."""
    A, hid, obs, _ = shape
    st, batch = regime_step(rid, shape, sk, bk, hp)
    new, out = sacd_update64(st, *batch, obs, hid, A, hp)
    assert np.isfinite(out["losses"]).all()
    for k in ("actor", "c1", "c2"):
        assert np.isfinite(out["grads"][k]).all() and np.isfinite(new[k]).all() and np.isfinite(new[k + "_v"]).all(), k
    assert np.isfinite(new["log_alpha"])
    compare_step(out["losses"], out["grads"], new, new, out, rid, hp)


def test_wide_regime_rows_find_batches():
    """The B = 4096 rows (their float64 updates take a while): finite, and clean_batch finds a batch."""
    for rid, shape, sk, bk, hp in ROWS:
        if shape[3] > 64:
            A, hid, obs, _ = shape
            st, batch = regime_step(rid, shape, sk, bk, hp)
            _, out = sacd_update64(st, *batch, obs, hid, A, hp)
            assert np.isfinite(out["losses"]).all() and all(np.isfinite(g).all() for g in out["grads"].values()), rid


# the row that shows each deviation, and the entry of the comparison it fails
CATCHES = {"no_eps": ("gap18.4-alpha5", "actor"), "ratio_one": ("gap18.4-alpha0.01", "actor"),
           "post_alpha": ("gap18.4-alpha5", "losses"), "no_shaping": ("gap12-alpha0.01", "losses"),
           "max_target": ("gap12-alpha0.01", "losses"), "stale_critics": ("gap12-alpha0.01", "losses"),
           "stale_soft": ("gap12-alpha0.01", "t1"), "no_target_entropy": ("gap12-alpha0.01", "losses")}


@pytest.mark.parametrize("mutant", MUTANTS)
def test_every_mutant_is_caught(mutant):
    rid, entry = CATCHES[mutant]
    (_, shape, sk, bk, hp), = [r for r in ROWS if r[0] == rid]
    st, batch = regime_step(rid, shape, sk, bk, hp)
    got = caught(st, batch, shape, hp, mutant)
    assert got is not None and got[1] == entry, (mutant, rid, got)
    if mutant in ("no_eps", "ratio_one"):                  # the worst entry: fc3 of the actor, where p is small
        A, hid, obs, _ = shape
        W, b = fc3(obs, hid, A)
        assert got[2] == "grad" and W.start <= got[4] < b.stop, got


def test_mutant_catches_over_all_rows():
    """Which rows see which deviation: each is seen by some row, and the +1e-8 deviations by the sharp rows only (a logit gap
    that puts some p near 1e-8 and alpha large enough for the entropy terms to matter)."""
    seen = {m: [] for m in MUTANTS}
    for rid, shape, sk, bk, hp in ROWS:
        if shape[3] > 64:
            continue
        st, batch = regime_step(rid, shape, sk, bk, hp)
        for m in MUTANTS:
            if caught(st, batch, shape, hp, m):
                seen[m].append(rid)
    assert all(seen.values()), {m: r for m, r in seen.items() if not r}
    for m in ("no_eps", "ratio_one"):
        assert not [r for r in seen[m] if r.startswith("gap12-alpha0.01")], (m, seen[m])
        assert "gap18.4-alpha5" in seen[m] and "gap120-alpha50" in seen[m], (m, seen[m])


def shape_sweep_rows():
    """test_sac_discrete_gpu.py's sweep_rows, with 'widest' resolved"""
    rows = [(27, 64, 100, B) for B in (1, 31, 32, 33, 64, 4096)]
    rows += [(2, 1, 4, 33), (31, 32, 128, 64), (2, 64, 100, 31), (31, 1, 100, 32), (27, 32, 4, 1), (2, 32, 128, 4096)]
    rows += [(A, WIDEST[A, obs], obs, 64) for A in (2, 27, 31) for obs in (4, 100, 128)]
    return rows


@pytest.mark.parametrize("mutant", ["no_eps", "ratio_one"])
def test_eps_mutants_pass_the_shape_sweep(mutant):
    """Both updates of every shape-sweep row, rebuilt from its seed (init_state, clean_batch, the float64 step standing in
    for the learner's state after the first): the deviation stays inside compare_step's bounds, so the sweep alone cannot
    see it."""
    for A, hid, obs, B in shape_sweep_rows():
        rng = np.random.default_rng(A * 1000 + obs + hid + B)
        st = init_state(rng, obs, hid, A)
        for step in range(2):
            batch = clean_batch(rng, st, B, obs, hid, A)
            assert caught(st, batch, (A, hid, obs, B), HP, mutant) is None, (mutant, A, hid, obs, B, step)
            st, _ = sacd_update64(st, *batch, obs, hid, A)


def test_fallback_needs_u_of_one():
    """u sum(p) in fp32 with u = nextafter(1, 0) stays below sum(p) for every sum of k equal fp32 probabilities 1/k (the
    product lies at least half an ulp below the sum, and exactly on a representable value when the sum is a power of two), so
    a Philox uniform never reaches the rounding fallback; a tape u of 1 does, and picks the last positive entry."""
    u = np.nextafter(np.float32(1), np.float32(0))
    for k in range(1, 32):
        for lead in (0, 3):
            p = np.zeros(lead + k + 4, np.float32)
            p[lead:lead + k] = np.float32(1) / np.float32(k)
            s = np.float32(0)
            for x in p:
                s = np.float32(s + x)
            assert np.float32(u * s) < s, k
            assert categorical_pick(p, u, np.float32) == categorical_pick(p, np.float32(1), np.float32) == lead + k - 1
            assert categorical_pick(p, np.float32(0), np.float32) == lead
