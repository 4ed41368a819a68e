"""Which network shape takes which kernel route: the tables the Q-network and SAC sweeps are parametrised over.

The learner accepts in_dim 1-128, 1-4 hidden layers of up to 128 units and 1-31 actions, and the host routes each shape to
one of several kernel variants.  The tensor-core act / TD kernel and training kernel come as a FIXED variant (compile-time
wgmma chains, wgmma.cuh mma_fixed) and a generic one (runtime k-step chains, 16-column tail chunks); shapes that do not fit
the training kernel get tensor-core TD targets feeding the fp32 update kernel, and shapes that do not fit the tensor-core
kernels at all run fp32 only.  SHAPES names the route each shape must take (pinned through Learner.route), so a shape that
silently moves to another route fails."""

# the four shipped Q-networks (in_dim, hidden, n_actions, dueling): QValue3 and QNet2 at hiden_dim 64, VAnet2, VAnet3
SHIPPED = [(100, [64, 64], 27, 0), (100, [64], 27, 0), (100, [64], 27, 1), (100, [128, 64], 27, 1)]

# (in_dim, hidden, n_actions, dueling, expected route): the route is (tensor-core act / TD kernel, tensor-core training
# kernel, forward tiles can reach 128 rows, training tiles can reach 64 rows, fp32 update kernel keeps both networks in
# shared memory).  The kernels' static shared memory counts against the 227 KB too: the last shape's tensor-core image fits
# only without it, and (32, [64, 64, 64]) trains in 32-row tiles for that reason.
SHAPES = [
    # generic forward + generic training kernel
    (100, [32], 27, 0, ("generic", "generic", True, True, True)),           # head over K = 32: 4 k-steps
    (100, [64, 32], 27, 1, ("generic", "generic", True, True, True)),       # 32-wide hidden layer into a dueling head
    (96, [64, 64], 27, 0, ("generic", "generic", False, True, True)),       # layer 0 over 12 k-steps
    (36, [64], 27, 0, ("generic", "generic", True, True, True)),            # layer 0 over 5 k-steps, in_dim padded to 40
    (12, [32, 32, 32, 32], 7, 1, ("generic", "generic", True, True, True)),  # 4 hidden layers: hm3 / hm4, dX over 5 layers
    (32, [64, 64, 64], 8, 0, ("generic", "generic", True, False, True)),    # 3 hidden layers of 64; 64-row training tiles do not fit
    (100, [20], 5, 0, ("generic", "generic", True, True, True)),            # 20 units padded to 32, 5 actions
    # FIXED forward + FIXED training kernel at shapes that are not shipped
    (100, [60], 27, 1, ("fixed", "fixed", True, True, True)),               # 4 zero units per 64
    (100, [64], 31, 1, ("fixed", "fixed", True, True, True)),               # V at head column 31
    (100, [64], 31, 0, ("fixed", "fixed", True, True, True)),               # every head column an action
    (124, [64], 27, 0, ("fixed", "fixed", False, True, True)),              # dW: 16 k-steps, ones column at row 124
    # tensor-core TD targets feeding the fp32 update kernel
    (100, [48], 27, 0, ("generic", None, True, False, True)),                # 32 + 16-column tail chunk
    (100, [112], 27, 0, ("generic", None, False, False, True)),              # 64 + 32 + 16-column tail chunk
    (128, [64], 27, 0, ("fixed", None, False, False, True)),                 # in_dim 128: no room for the dW ones column
    (100, [64, 64, 64], 27, 0, ("fixed", None, False, False, False)),        # training image too large; fp32 single-weights mode
    (64, [64, 64, 64, 64], 27, 1, ("fixed", None, False, False, False)),     # 4 hidden layers in the act / TD kernel
    # fp32 only
    (100, [128, 64, 64], 27, 1, (None, None, False, False, False)),          # VAnet4 at hiden_dim 64
    (99, [64], 27, 0, (None, None, False, False, True)),                     # in_dim % 4 != 0
    (12, [128, 64, 64], 27, 0, (None, None, False, False, True)),            # 64-row image fits only without the static smem
]


def pick(in_dim, hidden, n_actions, dueling):
    """The SHAPES row of a network."""
    return next(s for s in SHAPES if s[:4] == (in_dim, hidden, n_actions, dueling))


FIXED_SHIPPED = ("fixed", "fixed", True, True, True)
# one shape of every route in SHAPES, then the shipped 100-64-64-27 and VAnet2
ROUTES = [
    pick(100, [64, 32], 27, 1),          # generic forward + generic training, dueling head
    pick(96, [64, 64], 27, 0),           # generic, forward tiles stop at 64 rows
    pick(32, [64, 64, 64], 8, 0),        # generic, training tiles stop at 32 rows
    pick(100, [64], 31, 1),              # FIXED + FIXED, V at head column 31
    pick(124, [64], 27, 0),              # FIXED + FIXED, forward tiles stop at 64 rows
    pick(100, [48], 27, 0),              # tensor-core TD (16-column tail chunk) feeding the fp32 update
    pick(100, [112], 27, 0),             # the same, forward tiles stop at 64 rows
    pick(128, [64], 27, 0),              # FIXED TD feeding the fp32 update
    pick(100, [64, 64, 64], 27, 0),      # FIXED TD feeding the fp32 update in single-weights mode
    pick(100, [128, 64, 64], 27, 1),     # fp32 only, single weights, dueling
    pick(99, [64], 27, 0),               # fp32 only, in_dim % 4 != 0
    (100, [64, 64], 27, 0, ("fixed", "fixed", False, True, True)),   # shipped; its 128-row forward image does not fit
    (100, [64], 27, 1, FIXED_SHIPPED),
]
# B, algorithms: 32-row tiles with fused TD at NPRE = 1 and 2; bench.py's PER batch (32-row tiles, fused TD, 128 CTAs); 64-row
# tiles with fused TD; separate TD passes with 64 / 128-row forward tiles.  "ddqn" is the dueling trainer on a dueling head.
LEGS = {"B64-dqn": 64, "B64-ddqn": 64, "B4096-ddqn": 4096, "B6000-ddqn": 6000, "B12000-dqn": 12000}


def shape_id(s):
    """Test id of a SHAPES / ROUTES row: the network and its route."""
    in_dim, hidden, n_actions, dueling, (fwd, train, _, _, _) = s
    return "%d-%s-%d%s-fwd_%s-train_%s" % (in_dim, "x".join(map(str, hidden)), n_actions, "-duel" if dueling else "",
                                          fwd or "fp32", train or "fp32")


def net_id(s):
    """Test id of a network (in_dim, hidden, n_actions, dueling) without its route."""
    return "%d-%s-%d-%s" % (s[0], "x".join(map(str, s[1])), s[2], "duel" if s[3] else "q")


def act_sizes(route, n_sm):
    """1000 (32-row tiles), 64 n_sm + 37 (64-row tiles) and, where forward tiles reach 128 rows, 128 n_sm + 101."""
    return [1000, 64 * n_sm + 37] + ([128 * n_sm + 101] if route[2] else [])


def expected_route(route, n, n_sm, tc=True):
    fwd, train, fwd128, train64, dual = route if tc else (None, None, False, False, route[4])
    fwd_rows = None if fwd is None else 128 if (n >= 128 * n_sm and fwd128) else 64 if n >= 64 * n_sm else 32
    train_rows = None if train is None else 64 if (n > 32 * n_sm and train64) else 32
    return dict(tc_fwd=fwd, tc_train=train, fwd_rows=fwd_rows, train_rows=train_rows,
                td_fused=train is not None and -(-n // train_rows) <= n_sm, fp32_dual=dual)


# SAC (obs_dim, hidden, action_bound, accepted): hidden > 64 runs with the gradient-plane stride widened to round_up(hidden, 32)
SAC_SHAPES = [
    (100, 64, 1.0, True),       # shipped (config/Trainer.xml)
    (100, 64, 2.5, True),       # action_bound scales the action and the critics' action gradient
    (100, 32, 1.0, True),
    (100, 16, 1.0, True),
    (100, 50, 1.0, True),       # hidden % 4 != 0: zero pad columns in the backward planes
    (12, 17, 0.5, True),        # odd width: the transposed weights keep ld = out (ldw_of's odd branch)
    (124, 64, 1.0, True),       # largest obs_dim: critic input 126, padded by 2
    (60, 72, 1.0, True),        # hidden > 64: gradient planes of stride 96
    (8, 100, 1.0, True),        # hidden > 64: stride 128
    (4, 1, 1.0, True),          # width-1 edge
]


def sac_shape_id(sh):
    return "obs%d-h%d-bound%g" % sh[:3]
