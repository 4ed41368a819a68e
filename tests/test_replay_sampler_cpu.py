"""The replay sampler of the lockstep loops without a GPU: Philox4x32-10 against Random123's published vectors, the numpy
restatement (tests/replay_restatement.py) against csrc/replay.cuh and common.cuh compiled for the host, perm_index as a
bijection, and perm_index as a fair sampler: every stored transition, whatever its age, equally likely to be drawn, with no
excess or deficit of neighbouring pairs drawn together and consecutive epochs independent.  Also the paired store of the
host-driven path (Paired) against a plain FIFO list, and the update schedule on it (PairedLoop).

The statistics use fixed seeds and bounds chosen before the data: a chi-square p-value inside [1e-5, 1 - 1e-5] (too regular
is as wrong as biased) and |z| <= 4.5 for the pair and overlap counts."""
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy import stats

import replay_restatement as R
from conftest import ROOT

CSRC = os.path.join(ROOT, "dqn-based-uav-3d_path_planer_b200", "csrc")

# Random123 (Salmon et al. 2011) known-answer vectors of philox4x32_10: (ctr words, key words, output words)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


def kat_words(ctr, key):
    """(key, ctr_lo, ctr_hi) of Philox::gen for Random123's word order."""
    return key[0] | key[1] << 32, ctr[0] | ctr[1] << 32, ctr[2] | ctr[3] << 32


DRIVER = r"""
#include <cstdio>
#include <cstring>
#include "replay.cuh"
std::atomic<int> uavrl::g_pdl{1};
using namespace uavrl;
int main()
{
    char op[4];
    while (scanf("%3s", op) == 1) {
        if (!strcmp(op, "P")) {
            unsigned long long key, lo, hi; uint32_t out[4];
            scanf("%llu %llu %llu", &key, &lo, &hi);
            Philox::gen(key, lo, hi, out);
            printf("%u %u %u %u\n", out[0], out[1], out[2], out[3]);
        } else if (!strcmp(op, "T")) {
            unsigned long long key, salt; int g;
            scanf("%llu %llu %d", &key, &salt, &g);
            printf("%llu\n", (unsigned long long)trainer_key(key, salt, g));
        } else if (!strcmp(op, "Q")) {
            unsigned long long M, i0, n; uint32_t k[4];
            scanf("%llu %u %u %u %u %llu %llu", &M, &k[0], &k[1], &k[2], &k[3], &i0, &n);
            for (unsigned long long i = i0; i < i0 + n; ++i) printf("%llu ", (unsigned long long)perm_index(i, M, k));
            printf("\n");
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def header(tmp_path_factory):
    """Run the host-compiled header on a list of queries; returns one output line per query."""
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    d = tmp_path_factory.mktemp("replay_host")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    subprocess.check_call([nvcc, "-std=c++17", "-Xcompiler", "-Wall,-Werror,-Wno-unknown-pragmas", "-I", CSRC, str(src), "-o", str(exe)])

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return out.splitlines()
    return run


def test_philox_known_answers(header):
    lines = header(["P %d %d %d" % kat_words(c, k) for c, k, _ in KAT])
    for (ctr, key, want), line in zip(KAT, lines):
        assert tuple(int(x) for x in R.philox(*kat_words(ctr, key))) == want
        assert tuple(int(x) for x in line.split()) == want


def test_philox_and_trainer_key_match_header(header):
    rng = np.random.default_rng(1)
    q = [tuple(int(x) for x in rng.integers(0, 1 << 63, 3, dtype=np.uint64) * 2 + rng.integers(0, 2, 3, dtype=np.uint64))
         for _ in range(200)]
    for (key, lo, hi), line in zip(q, header(["P %d %d %d" % t for t in q])):
        assert [int(x) for x in R.philox(key, lo, hi)] == [int(x) for x in line.split()]
    salts = (R.K_ACT_SALT, R.K_SAMPLE_SALT, R.K_FED_SALT, R.K_PER_SALT)
    tq = [(key, s, g) for (key, _, _) in q[:20] for s in salts for g in (0, 1, 2, 7)] + [(R.M64, R.K_SAMPLE_SALT, 3)]
    for (key, s, g), line in zip(tq, header(["T %d %d %d" % t for t in tq])):
        assert R.trainer_key(key, s, g) == int(line)
    assert R.trainer_key(5 ^ R.K_SAMPLE_SALT, R.K_SAMPLE_SALT, 3) == 8 ^ R.K_SAMPLE_SALT       # trainer g = seed + g


def edge_sizes():
    """M = 2, 3 and 2^k - 1, 2^k, 2^k + 1 for k = 2..21 (odd and even bit counts: odd ones walk a domain up to 4 M), plus
    the benchmark's largest ring: 128 frames x 8 192 envs."""
    out = {2, 3}
    for k in range(2, 22):
        out |= {(1 << k) - 1, 1 << k, (1 << k) + 1}
    return sorted(out) + [128 * 8192, 128 * 8192 - 8192]


def test_perm_index_matches_header(header):
    rng = np.random.default_rng(2)
    q = []
    for M in edge_sizes():
        for _ in range(3):
            k = rng.integers(0, 1 << 32, 4, dtype=np.uint64)
            n = min(M, 300)
            i0 = int(rng.integers(0, M - n + 1))
            q.append((M, k, i0, n))
    lines = header(["Q %d %d %d %d %d %d %d" % (M, *map(int, k), i0, n) for M, k, i0, n in q])
    for (M, k, i0, n), line in zip(q, lines):
        got = np.array([int(x) for x in line.split()], np.uint64)
        assert np.array_equal(got, R.perm_index(np.arange(i0, i0 + n), M, k)), (M, i0)
    # keys as the loops form them: Philox of (seed ^ salt, epoch, 0x5A17), trainer keys included
    q = [(M, R.sample_key(seed, ep, g)) for M in (3840, 65, 1 << 20) for seed in (1, 42) for ep in (1, 2, 1000) for g in (0, 2)]
    lines = header(["Q %d %d %d %d %d 0 64" % (M, *map(int, k)) for M, k in q])
    for (M, k), line in zip(q, lines):
        assert [int(x) for x in line.split()] == [int(x) for x in R.perm_index(np.arange(64), M, k)]


def test_perm_index_is_a_bijection():
    rng = np.random.default_rng(3)
    sizes = list(range(1, 4097)) + [int(x) for x in rng.integers(4097, 1 << 20, 12)] + [(1 << 18) + 1, 128 * 8192]
    for M in sizes:
        k = rng.integers(0, 1 << 32, 4, dtype=np.uint64)
        p = R.perm_index(np.arange(M), M, k)
        assert p.max() < M and np.unique(p).size == M, M


def test_walk_domain_sizes():
    """An odd bit count runs the Feistel network on bits + 1 bits: cycle walking covers up to 4 M."""
    assert R.perm_bits(2) == (1, 1) and R.perm_bits(3) == (2, 1) and R.perm_bits(5) == (3, 2)
    assert R.perm_bits(1 << 20) == (20, 10) and R.perm_bits((1 << 20) + 1) == (21, 11)


# ------------------------------------------------------------------ fairness
def two_sided(p):
    assert 1e-5 <= p <= 1 - 1e-5, p


def inclusion_chi2(counts, E, B, M):
    """Per-cell inclusion counts over E epochs of B draws without replacement from M: each is a sum of E independent
    Bernoulli(B / M); sum of squared standardised deviations ~ chi-square with M - 1 degrees of freedom after the M / (M - 1)
    correction for the fixed total."""
    p = B / M
    chi = float((((counts - E * p) ** 2) / (E * p * (1 - p))).sum()) * (M - 1) / M
    return stats.chi2.sf(chi, M - 1), chi / (M - 1)


# (M, B, epochs, envs per frame): B / M from 1/60 to (M - 1) / M; odd and even bit counts
FAIR = [
    (65, 64, 20000, 13),             # B = M - 1
    (3840, 64, 100000, 64),          # 60 frames of 64 envs, B / M = 1/60
    (1536, 1024, 8000, 512),         # 3 frames of 512
    (12288, 6144, 1000, 2048),       # 6 frames, B / M = 1/2
    ((1 << 17) + 1, 4096, 2000, 1),  # 18 bits: a 2^18 Feistel domain walked
]


@pytest.mark.parametrize("M,B,E,Ng", FAIR, ids=["M%d-B%d" % c[:2] for c in FAIR])
def test_perm_index_is_a_fair_sample(M, B, E, Ng):
    S = R.sample(7 + M, np.arange(1, E + 1), M, B)
    assert S.shape == (E, B)
    # every transition equally likely
    c = np.bincount(S.ravel(), minlength=M)
    p, ratio = inclusion_chi2(c, E, B, M)
    two_sided(p)
    # ... whatever its age: cells of one frame (the logical order is age, oldest first)
    if Ng > 1 and M % Ng == 0:
        F = M // Ng
        cf = c.reshape(F, Ng).sum(1)
        q = Ng / M                                             # hypergeometric draws per epoch from one frame's cells
        var = E * B * q * (1 - q) * (M - B) / (M - 1)
        chi = float(((cf - E * B * q) ** 2 / var).sum()) * (F - 1) / F
        two_sided(stats.chi2.sf(chi, F - 1))
    # pairs drawn together: (same env, adjacent frames), (same frame, adjacent envs), against the hypergeometric rate
    inc = np.zeros((E, M), bool)
    np.put_along_axis(inc, S, True, axis=1)
    pair_p = B * (B - 1) / (M * (M - 1))
    pairs = {}
    if Ng < M:
        pairs["frames"] = inc[:, :-Ng] & inc[:, Ng:]
    if Ng > 1:
        e = np.arange(M - 1)
        pairs["envs"] = (inc[:, :-1] & inc[:, 1:])[:, (e % Ng) != Ng - 1]
    pairs["any"] = inc[:, :-1] & inc[:, 1:]
    for name, m in pairs.items():
        per_epoch = m.sum(1).astype(np.float64)
        z = (per_epoch.mean() - m.shape[1] * pair_p) / (per_epoch.std() / np.sqrt(E) + 1e-300)
        assert abs(z) <= 4.5, (name, z, per_epoch.mean(), m.shape[1] * pair_p)
    # consecutive epochs: overlap B^2 / M with the hypergeometric spread
    ov = (inc[1:] & inc[:-1]).sum(1).astype(np.float64)
    mean = B * B / M
    var = B * (B / M) * (1 - B / M) * (M - B) / (M - 1)
    if var > 0:
        z = (ov.mean() - mean) / np.sqrt(var / ov.size)
        assert abs(z) <= 4.5, (z, ov.mean(), mean)


def test_loop_epochs_draw_distinct_batches():
    """Each epoch's batch holds B distinct indices, and batch position b is not tied to one index: over 5 000 epochs of the
    first ring size test_perm_index_is_a_fair_sample covers, position 0 visits every index."""
    S = R.sample(11, np.arange(1, 5001), 65, 64)
    assert all(np.unique(row).size == 64 for row in S)
    assert np.unique(S[:, 0]).size == 65
    S = R.sample(11, np.arange(1, 2001), 3840, 64)
    two_sided(stats.chisquare(np.bincount(S[:, 0] // 64, minlength=60)).pvalue)


# ------------------------------------------------------------------ the ring and the loop schedule
def test_ring_arithmetic():
    ring = R.Ring(capacity=3 * 96, n_envs=96, trainers=3)
    assert ring.ring_frames == 4 and ring.Ng == 32
    seen = []
    for k in range(1, 10):
        ring.commit()
        assert ring.count == min(k, 3) * 96 and ring.head == k % 4
        assert ring.oldest() == (k - min(k, 3)) % 4
        seen.append(ring.oldest())
        J = ring.newest()
        slot, row, row2, fresh = ring.ref(J)
        assert np.array_equal(slot // 96, np.full(96, (k - 1) % 4)) and fresh.all() and np.array_equal(row2 // 96, np.full(96, k % 4))
        _, _, _, fresh_all = ring.ref(np.arange(ring.count))
        assert fresh_all.sum() == 96                             # only the newest group's next states are fresh
    assert seen == [0, 0, 0, 1, 2, 3, 0, 1, 2]
    # trainer g's local index j -> the whole-ring index of env g Ng + j mod Ng in frame j // Ng
    j = np.arange(ring.count_g())
    for g in range(3):
        J = ring.logical(j, g)
        assert np.array_equal(J % 96 // 32, np.full(j.size, g)) and np.array_equal(J // 96, j // 32)


def test_loop_schedule():
    """B = 64, N = 48, 2 trainers: the skip rule counts per trainer; the epoch counts every update, sampled or not."""
    loop = R.Loop(R.Ring(48 * 8, 48, 2), seed=5, batch_size=64, update_loop=3)
    its = [loop.iteration(1) for _ in range(6)]
    assert [u[0] is None for u in its] == [True, True, False, False, False, False]   # 24, 48, 72 > 64 per trainer
    assert [u[0][0] for u in its[2:]] == [3, 4, 5, 6] and [u[0][2] for u in its[2:]] == [True, False, False, True]
    assert loop.adam_t == 4 and loop.act_calls == 6 and loop.epoch == 6
    e, idx, _ = its[2][0]
    assert np.array_equal(idx[1], R.sample(5 + 1, e, 72, 64)) and not np.array_equal(idx[0], idx[1])


# ------------------------------------------------------------------ the paired store of the host-driven path
def paired_pushes(rng, cap, total):
    """Ragged push sizes summing to at least `total`: single transitions, pushes larger than what is left before the wrap, and
    pushes of exactly the capacity."""
    out, done = [], 0
    while done < total:
        k = int(rng.integers(0, 4))
        left = cap - (done % cap)
        n = [1, int(rng.integers(1, cap + 1)), cap, min(cap, left + int(rng.integers(1, cap + 1)))][k]
        out.append(n)
        done += n
    return out


@pytest.mark.parametrize("cap", [1, 2, 7, 64, 1000])
def test_paired_store_is_a_fifo(cap):
    """Paired against a plain FIFO list: after every ragged push, logical index j (0 = oldest) names the slot that holds the
    FIFO's j-th transition, oldest / count / head agree, and the newest indices are the last push in order."""
    rng = np.random.default_rng(cap)
    P = R.Paired(cap)
    fifo, held = [], {}                   # transition ids oldest first; slot -> id it holds
    nxt = 0
    for n in paired_pushes(rng, cap, 6 * cap + 5):
        ids = list(range(nxt, nxt + n))
        nxt += n
        slots = P.push(n)
        assert slots.shape == (n,) and ((0 <= slots) & (slots < cap)).all()
        for i, s in zip(ids, slots):
            held[int(s)] = i
        fifo = (fifo + ids)[-cap:]
        assert P.count == len(fifo) and P.head == nxt % cap
        j = np.arange(P.count)
        assert [held[int(s)] for s in P.slot(j)] == fifo
        assert np.array_equal(P.logical(P.slot(j)), j)
        assert [held[int(s)] for s in P.slot(P.newest(min(n, cap)))] == ids[-cap:]
        assert P.oldest() == (0 if nxt <= cap else nxt % cap)


def test_paired_schedule():
    """B = 5 on a 9-slot store: the epoch counts every call; count <= B samples nothing; adam_t counts real updates; the hard
    update lands on epochs divisible by update_loop; the draw is sample(seed, epoch, count, B)."""
    P = R.Paired(9)
    loop = R.PairedLoop(P, seed=3, batch_size=5, update_loop=3)
    got = []
    for n in (2, 3, 1, 9, 4):             # count 2, 5 (= B), 6 (= B + 1), 9 (full), 9 (wrapped)
        P.push(n)
        got.append(loop.update())
    assert [u is None for u in got] == [True, True, False, False, False]
    assert [u[0] for u in got[2:]] == [3, 4, 5] and [u[2] for u in got[2:]] == [True, False, False]
    assert loop.epoch == 5 and loop.adam_t == 3
    assert np.array_equal(got[2][1], R.sample(3, 3, 6, 5)) and np.array_equal(got[4][1], R.sample(3, 5, 9, 5))
