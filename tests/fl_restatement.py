"""A numpy restatement of the selective federated aggregation (Envs/PathPlan_City.py:644-684,
Federated_Learning_choice) that the federation tests judge the device against.

Round p = 0, 1, ..., G-1, in place: the Q-values of trainer p on its probe states, the mean squared difference to
every other trainer's current Q-values on the same states (float64 here), a stable sort by loss, the first
k = (G - 1) // 2 trainers kept, and trainer p's parameters replaced by the float32 in-order sum
theta_p + theta_c0 + theta_c1 + ... divided once by k + 1.  Only q_local changes.  check_rounds holds the device's rounds to
it.  federate_actors restates the actor aggregation of the SAC trainers (Federated_Learning_AC)."""
import numpy as np

from qnet_restatement import f64_forward, f64_unpack, net_layers


def q64(theta, x, net):
    """Q-values [n, A] in float64 of one flat parameter vector of net = (in_dim, hidden, n_actions, dueling)."""
    return f64_forward(f64_unpack(net_layers(*net), theta), net[3], x)[0]


def average(theta, p, chosen):
    """float32 theta_p + theta_c0 + ... (left to right), then one division by len(chosen) + 1."""
    s = theta[p].astype(np.float32).copy()
    for c in chosen:
        s = (s + theta[c]).astype(np.float32)
    return (s / np.float32(len(chosen) + 1)).astype(np.float32)


def round_losses(cur, p, probes_p, net):
    """float64 losses of round p against the parameters `cur` ([p][p] = 0)."""
    G = cur.shape[0]
    own = q64(cur[p], probes_p, net)
    m = np.zeros(G)
    for q in range(G):
        if q != p:
            m[q] = np.mean((own - q64(cur[q], probes_p, net)) ** 2)
    return m


def rank(m, p):
    """The reference's selection: trainers q != p sorted by (loss, q), the first (G - 1) // 2."""
    G = m.size
    order = sorted((q for q in range(G) if q != p), key=lambda q: m[q])      # stable: equal losses keep ascending q
    return order[:(G - 1) // 2]


def federate(local0, probes, in_dim, hidden, n_actions, dueling, jacobi=False, chosen_given=None):
    """Returns (parameters after, chosen [G][max(1, k)] (-1 padded), float64 losses [G][G]).
    jacobi = True: every loss and every average from the initial parameters (the wrong round order)."""
    net = (in_dim, list(hidden), n_actions, bool(dueling))
    theta = np.array(local0, np.float32, copy=True)
    G = theta.shape[0]
    k = (G - 1) // 2
    chosen = np.full((G, max(1, k)), -1, np.int64)
    M = np.zeros((G, G))
    for p in range(G):
        src = local0 if jacobi else theta
        M[p] = round_losses(src, p, probes[p], net)
        ch = list(chosen_given[p][:k]) if chosen_given is not None else rank(M[p], p)
        chosen[p, :k] = ch
        theta[p] = average(src, p, ch)
    return theta, chosen, M


def net_of(shape):
    in_dim, hidden, nA, dueling = shape
    return (in_dim, list(hidden), nA, bool(dueling))


def magnitude(theta, x, net):
    """|Q| bound per row and action: the forward with |W|, |b| and |x| (ReLU never increases a magnitude)."""
    in_dim, hidden, nA, dueling = net
    h = np.abs(np.asarray(x, np.float64))
    blocks = [(np.abs(W), np.abs(b)) for W, b in f64_unpack(net_layers(*net), theta)]
    for W, b in blocks[:len(hidden)]:
        h = h @ W.T + b
    A = h @ blocks[len(hidden)][0].T + blocks[len(hidden)][1]
    if dueling:
        V = h @ blocks[len(hidden) + 1][0].T + blocks[len(hidden) + 1][1]
        A = V + 2 * A.max(axis=1, keepdims=True) + A
    return A


def check_rounds(before, after, probes, losses, chosen, shape, rounds):
    """The device's rounds `rounds` (before / after: the parameters [G][P] around the call; losses, chosen: what it reported),
    each on its own: round p is fully determined by the final parameters of the trainers q < p, the initial parameters of
    the trainers q > p and its probes.  Float64 losses within a magnitude bound, a selection that is the (loss, index)-sorted
    prefix up to float64 near-ties, and theta_p bit for bit the float32 in-order average of the selection the device made."""
    net = net_of(shape)
    G = before.shape[0]
    k = (G - 1) // 2
    gamma = 8e-6 * (len(net[1]) + 1)                      # fp32-grade forward: relative error per layer of the magnitude chain
    for p in rounds:
        cur = np.concatenate([after[:p], before[p:]])
        x = probes[p]
        own = q64(cur[p], x, net)
        mag_p = magnitude(cur[p], x, net)
        m64, tol = np.zeros(G), np.zeros(G)
        for q in range(G):
            if q == p:
                continue
            Qq = q64(cur[q], x, net)
            d = own - Qq
            m64[q] = np.mean(d * d)
            delta = gamma * (mag_p + magnitude(cur[q], x, net))
            tol[q] = np.mean(2 * np.abs(d) * delta + delta * delta) + 1e-6 * m64[q] + 1e-30
        got = losses[p].astype(np.float64)
        assert got[p] == 0.0
        bad = np.abs(got - m64) > tol
        assert not bad.any(), (p, np.nonzero(bad)[0][:5], got[bad][:5], m64[bad][:5], tol[bad][:5])
        if k == 0:
            assert (chosen[p] == -1).all()
            assert np.array_equal(after[p], before[p])
            continue
        c = [int(v) for v in chosen[p][:k]]
        assert len(set(c)) == k and p not in c and all(0 <= v < G for v in c), (p, c)
        # the device's own ranking: (loss, index) order along the chosen list
        for a, b in zip(c, c[1:]):
            assert (got[a], a) < (got[b], b), (p, c)
        # against float64: a chosen trainer may only beat an unchosen one it lies within the bounds of
        rest = [q for q in range(G) if q != p and q not in c]
        if rest:
            worst = max(c, key=lambda q: m64[q] - tol[q])
            best = min(rest, key=lambda q: m64[q] + tol[q])
            assert m64[worst] - tol[worst] <= m64[best] + tol[best], (p, worst, best)
            ref = rank(m64, p)
            for q in set(c) ^ set(ref):
                others = [r for r in (set(c) | set(ref)) if r != q]
                assert any(abs(m64[q] - m64[r]) <= tol[q] + tol[r] for r in others), (p, q)
        assert np.array_equal(after[p], average(cur, p, c)), "round %d: theta_p is not the in-order float32 average" % p


def federate_actors(actors):
    """Every actor <- the float32 sum theta_0 + theta_1 + ... + theta_{G-1}, added left to right in trainer order.  The
    reference's division by G assigns into a temporary state_dict and is lost, so nothing is divided."""
    actors = np.asarray(actors, np.float32)
    s = actors[0].copy()
    for g in range(1, actors.shape[0]):
        s = np.add(s, actors[g], dtype=np.float32)
    return np.broadcast_to(s, actors.shape).copy()
