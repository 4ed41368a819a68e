"""A numpy restatement of the selective federated aggregation (Envs/PathPlan_City.py:644-684,
Federated_Learning_choice) that the federation tests judge the device against.

Round p = 0, 1, ..., G-1, in place: the Q-values of trainer p on its probe states, the mean squared difference to
every other trainer's current Q-values on the same states (float64 here), a stable sort by loss, the first
k = (G - 1) // 2 trainers kept, and trainer p's parameters replaced by the float32 in-order sum
theta_p + theta_c0 + theta_c1 + ... divided once by k + 1.  Only q_local changes."""
import numpy as np


def layers(in_dim, hidden, n_actions, dueling):
    """(rows, cols) of every weight block in the flat state_dict order, each followed by its bias."""
    out, fan = [], in_dim
    for h in hidden:
        out.append((h, fan))
        fan = h
    out.append((n_actions, fan))
    if dueling:
        out.append((1, fan))
    return out


def forward64(theta, x, in_dim, hidden, n_actions, dueling):
    """Q-values [n, A] in float64 of one flat parameter vector."""
    off, h = 0, np.asarray(x, np.float64)
    blocks = []
    for r, c in layers(in_dim, hidden, n_actions, dueling):
        W = np.asarray(theta[off:off + r * c], np.float64).reshape(r, c); off += r * c
        b = np.asarray(theta[off:off + r], np.float64); off += r
        blocks.append((W, b))
    assert off == theta.size
    for W, b in blocks[:len(hidden)]:
        h = np.maximum(h @ W.T + b, 0.0)
    WA, bA = blocks[len(hidden)]
    A = h @ WA.T + bA
    if not dueling:
        return A
    WV, bV = blocks[len(hidden) + 1]
    V = h @ WV.T + bV
    return V + A - A.mean(axis=1, keepdims=True)


def average(theta, p, chosen):
    """float32 theta_p + theta_c0 + ... (left to right), then one division by len(chosen) + 1."""
    s = theta[p].astype(np.float32).copy()
    for c in chosen:
        s = (s + theta[c]).astype(np.float32)
    return (s / np.float32(len(chosen) + 1)).astype(np.float32)


def round_losses(cur, p, probes_p, net):
    """float64 losses of round p against the parameters `cur` ([p][p] = 0)."""
    G = cur.shape[0]
    own = forward64(cur[p], probes_p, *net)
    m = np.zeros(G)
    for q in range(G):
        if q != p:
            m[q] = np.mean((own - forward64(cur[q], probes_p, *net)) ** 2)
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
