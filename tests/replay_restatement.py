"""A numpy restatement of the replay sampler the lockstep loops draw their batches with (csrc/replay.cuh, replay.cu, common.cuh,
learner.cuh, sac.cu), which the sampler tests judge the device against.

Philox4x32-10 keyed by (seed, salt, trainer); the keyed permutation perm_index (4-round Feistel with cycle walking) that turns
batch position b into the b-th of B distinct trainer-local replay indices; the lockstep ring (frames of N envs, trainer g owning
envs [g Ng, (g + 1) Ng)) that maps such an index to a whole-ring logical index; the loop's schedule (an epoch per update,
nothing sampled while a trainer holds <= batch_size transitions, a hard target update every update_loop-th epoch); the paired
store of the host-driven path (lockstep_envs = 0) and the same schedule on it; the eps-greedy draw of the act pass, the
prioritised sampler's uniforms and SAC's Box-Muller reparameterisation noise."""
import numpy as np

M64 = (1 << 64) - 1
K_ACT_SALT, K_SAMPLE_SALT, K_FED_SALT, K_PER_SALT = 0xAC7, 0x5EED, 0xFED, 0x9E12
K_NOISE_SALT = 0x5AC5                 # sac.cu kNoiseSalt
SAMPLE_STREAM = 0x5A17                # the high counter word of the sampling key draw
SAC_ACT_CTR = 1 << 63                 # sac.cu: get_action's noise counter is this bit | the act call


def trainer_key(key, salt, g):
    """Trainer g of a grouped learner draws what a stand-alone learner seeded with seed + g draws."""
    return (((key ^ salt) + g) & M64) ^ salt


# ------------------------------------------------------------------ Philox4x32-10
def philox(key, ctr_lo, ctr_hi):
    """Philox4x32-10 of 64-bit key and counter words (arrays broadcast): uint32 array [..., 4]."""
    key, ctr_lo, ctr_hi = (np.asarray(x, np.uint64) for x in (key, ctr_lo, ctr_hi))
    key, ctr_lo, ctr_hi = np.broadcast_arrays(key, ctr_lo, ctr_hi)
    m32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    c = [ctr_lo & m32, ctr_lo >> s32, ctr_hi & m32, ctr_hi >> s32]
    k0, k1 = key & m32, key >> s32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> s32) ^ c[1] ^ k0, p1 & m32, (p0 >> s32) ^ c[3] ^ k1, p0 & m32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return np.stack(c, -1).astype(np.uint32)


def u01(x):
    """Philox::u01: 24 random bits as a float32 in [0, 1)."""
    return ((np.asarray(x, np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


# ------------------------------------------------------------------ the keyed permutation
def mix32(x):
    x = np.asarray(x, np.uint64) & np.uint64(0xFFFFFFFF)
    m = np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16); x = (x * np.uint64(0x7FEB352D)) & m
    x ^= x >> np.uint64(15); x = (x * np.uint64(0x846CA68B)) & m
    x ^= x >> np.uint64(16)
    return x


def perm_bits(M):
    """(bits, h): the Feistel network runs on 2 h bits, h = ceil(bits / 2), 2^bits >= M."""
    bits = 1
    while (1 << bits) < M:
        bits += 1
    return bits, (bits + 1) // 2


def perm_index(i, M, key4):
    """Elements i (array) of the keyed permutation of [0, M); key4 = the 4 uint32 words of the sampling draw ([4], or
    [..., 4] broadcasting against i: one permutation per element)."""
    _, h = perm_bits(int(M))
    mask = np.uint64((1 << h) - 1)
    hs = np.uint64(h)
    x, K = np.broadcast_arrays(np.array(i, np.uint64, ndmin=1)[..., None], np.asarray(key4, np.uint64))
    x, K = x[..., 0].copy(), K.reshape(-1, 4)
    flat = x.reshape(-1)
    todo = np.arange(flat.size)
    while todo.size:
        L, R = (flat[todo] >> hs) & mask, flat[todo] & mask
        for r in range(4):
            f = mix32(R ^ K[todo, r]) & mask
            L, R = R, L ^ f
        flat[todo] = (L << hs) | R
        todo = todo[flat[todo] >= np.uint64(M)]
    return flat.reshape(x.shape)


def sample_key(seed, epoch, g=0):
    """The 4 key words of the permutation trainer g draws at epoch `epoch` (replay.cu source, trainer_src)."""
    key = (seed ^ K_SAMPLE_SALT) & M64
    if g:
        key = trainer_key(key, K_SAMPLE_SALT, g)
    return philox(key, epoch, SAMPLE_STREAM)


def sample(seed, epoch, count, B, g=0):
    """The trainer-local logical indices (0 = oldest) that update `epoch` of trainer g draws from its `count` transitions;
    epoch may be an array of E epochs: [E, B]."""
    key = sample_key(seed, np.asarray(epoch), g)
    return perm_index(np.arange(B), count, key[..., None, :]).astype(np.int64)


# ------------------------------------------------------------------ the lockstep ring
class Ring:
    """ReplayStore in its lockstep layout: ring_frames frames of N envs, G trainers of Ng = N / G envs each."""

    def __init__(self, capacity, n_envs, trainers=1):
        self.N, self.G = n_envs, trainers
        self.Ng = n_envs // trainers
        cap_frames = max(2, -(-(capacity // trainers) // self.Ng))
        self.ring_frames = cap_frames + 1
        self.head = 0
        self.count = 0

    def commit(self):
        self.head = (self.head + 1) % self.ring_frames
        self.count = min(self.count + self.N, (self.ring_frames - 1) * self.N)

    def oldest(self):
        return (self.head - self.count // self.N) % self.ring_frames

    def count_g(self):
        return self.count // self.G

    def logical(self, j, g=0):
        """Trainer g's local index j -> the whole-ring logical index (gather's argument)."""
        j = np.asarray(j, np.int64)
        return (j // self.Ng) * self.N + g * self.Ng + j % self.Ng

    def ref(self, J):
        """Whole-ring logical index -> (slot, row, row2, fresh): replay_ref; fresh = the next-state row lies in the frame
        the current iteration's env step writes."""
        J = np.asarray(J, np.int64)
        f = (self.oldest() + J // self.N) % self.ring_frames
        e = J % self.N
        f2 = (f + 1) % self.ring_frames
        return f * self.N + e, f * self.N + e, f2 * self.N + e, f2 == self.head

    def newest(self):
        """Whole-ring logical indices of the transition group the last commit made (iteration order of the envs)."""
        return np.arange(self.count - self.N, self.count)


class Loop:
    """The counters of a lockstep learner and its ring, advanced as uavrl_train_run / uavrl_sac_train_run advance them.
    iteration() returns the updates of one iteration: (epoch, per-trainer local indices, hard target update) or None for an
    update skipped because a trainer holds <= batch_size transitions (the epoch counts either way)."""

    def __init__(self, ring, seed, batch_size, update_loop=0, epoch=0, act_calls=0):
        self.ring, self.seed, self.B, self.update_loop = ring, seed, batch_size, update_loop
        self.epoch, self.act_calls, self.adam_t = epoch, act_calls, 0

    def iteration(self, updates_per_iter=1):
        self.act_calls += 1
        self.ring.commit()
        out = []
        for _ in range(updates_per_iter):
            self.epoch += 1
            if self.ring.count_g() <= self.B:
                out.append(None)
                continue
            self.adam_t += 1
            idx = [sample(self.seed, self.epoch, self.ring.count_g(), self.B, g) for g in range(self.ring.G)]
            hard = self.update_loop > 0 and self.epoch % self.update_loop == 0
            out.append((self.epoch, idx, hard))
        return out


# ------------------------------------------------------------------ the paired store
class Paired:
    """ReplayStore in its paired layout (lockstep_envs = 0): a FIFO of `capacity` slots that uavrl_replay_push fills; head = the
    next slot written, count = the valid transitions, logical index j (0 = oldest) in slot (oldest + j) mod capacity."""

    def __init__(self, capacity):
        self.slots = capacity
        self.head = 0
        self.count = 0

    def push(self, n):
        """n new transitions (1 <= n <= capacity; the push may wrap): the slots they land in, in push order."""
        assert 1 <= n <= self.slots
        out = (self.head + np.arange(n)) % self.slots
        self.head = (self.head + n) % self.slots
        self.count = min(self.count + n, self.slots)
        return out

    def oldest(self):
        return (self.head - self.count) % self.slots

    def slot(self, j):
        """Logical index j -> slot (gather's mapping)."""
        return (self.oldest() + np.asarray(j, np.int64)) % self.slots

    def logical(self, slot):
        return (np.asarray(slot, np.int64) - self.oldest()) % self.slots

    def newest(self, n):
        """Logical indices of the last n transitions pushed, in push order."""
        return np.arange(self.count - n, self.count)


class PairedLoop:
    """The counters of a learner on a paired store as update() / learn_off_policy advance them: the epoch counts every call,
    nothing is sampled while count <= batch_size, adam_t counts real updates only, and an update whose epoch is a multiple of
    update_loop ends with the hard target update.  update() returns (epoch, logical indices, hard) or None for a skipped
    call."""

    def __init__(self, store, seed, batch_size, update_loop=0, epoch=0, adam_t=0):
        self.store, self.seed, self.B, self.update_loop = store, seed, batch_size, update_loop
        self.epoch, self.adam_t = epoch, adam_t

    def update(self):
        self.epoch += 1
        if self.store.count <= self.B:
            return None
        self.adam_t += 1
        hard = self.update_loop > 0 and self.epoch % self.update_loop == 0
        return self.epoch, sample(self.seed, self.epoch, self.store.count, self.B), hard


# ------------------------------------------------------------------ the act pass and SAC's noise
def eps_greedy(seed, call, n_rows, eps, n_actions, g=0):
    """learner.cuh eps_greedy without tapes for rows 0..n_rows-1 of trainer g at act call `call`: (greedy mask, random action)."""
    key = trainer_key((seed ^ K_ACT_SALT) & M64, K_ACT_SALT, g) if g else (seed ^ K_ACT_SALT) & M64
    r = philox(key, call, np.arange(n_rows, dtype=np.uint64))
    u = u01(r[:, 0])
    ra = ((r[:, 1].astype(np.uint64) * np.uint64(n_actions)) >> np.uint64(32)).astype(np.int32)
    return u > np.float32(eps), ra


def per_uniforms(seed, call, B):
    """per.cu per_sample_kernel without a u-tape: the B uniforms in [0, 1) (53 random bits) of sampling call `call` of a
    stand-alone learner."""
    r = philox((seed ^ K_PER_SALT) & M64, call, np.arange(B, dtype=np.uint64)).astype(np.uint64)
    bits = ((r[:, 0] >> np.uint64(5)) << np.uint64(26)) | (r[:, 1] >> np.uint64(6))
    return bits.astype(np.float64) * (1.0 / 9007199254740992.0)


def sac_noise(seed, ctr, n_rows, g=0):
    """sac.cu noise2 for rows 0..n_rows-1 of trainer g: [n_rows, 2] float64 standard normals (Box-Muller evaluated in float64 on
    the float32 uniforms the kernel forms; the kernel's logf / cospif / sinpif differ from it by a few ulp)."""
    key = trainer_key((seed ^ K_NOISE_SALT) & M64, K_NOISE_SALT, g)
    r = philox(key, ctr, np.arange(n_rows, dtype=np.uint64))
    u0 = ((r[:, 0] >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)
    u1 = u01(r[:, 1])
    rad = np.sqrt(-2.0 * np.log(u0.astype(np.float64)))
    ang = 2.0 * np.pi * u1.astype(np.float64)
    return np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)


def sac_update_ctrs(epoch):
    """The noise counters of SAC update `epoch`: the TD target's next-state actions, then the actor leg's actions."""
    return 2 * epoch, 2 * epoch + 1
