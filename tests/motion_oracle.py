"""The moving-obstacle rule (include/uavrl.h, uavrl_env_set_motion) on top of the CPU oracle: one obstacle table shared by an
OracleBatch, advanced once per step.  The oracle reads its city's cylinder table and its APF velocities through pointers, so
the table is written into those arrays in place: the step runs on O_t, then every obstacle runs, then the observation is taken
on O_{t+1}."""
import hashlib

import numpy as np

import oracle as O


def table_digest(tab):
    """16-byte BLAKE2b of a table's rows (x, y, vx, vy) as fp64: equal digests mean bit-identical tables."""
    return hashlib.blake2b(np.ascontiguousarray(tab, np.float64).tobytes(), digest_size=16).digest()


def velocity_signs(tab):
    """Per row: bit 0 = vx < 0, bit 1 = vy < 0."""
    tab = np.asarray(tab, np.float64)
    return ((tab[:, 2] < 0).astype(np.uint8) | ((tab[:, 3] < 0).astype(np.uint8) << 1))


def wall_reflections(before, after):
    """Reflections per wall between two tables of the same rows (any number of runs apart, one reflection per row at most):
    at x = 0 vx turns from negative to positive, at x = len from positive to negative; likewise y at 0 and width."""
    b, a = np.asarray(before, np.float64), np.asarray(after, np.float64)
    return {"x0": int(((b[:, 2] < 0) & (a[:, 2] > 0)).sum()), "xlen": int(((b[:, 2] > 0) & (a[:, 2] < 0)).sum()),
            "y0": int(((b[:, 3] < 0) & (a[:, 3] > 0)).sum()), "ywidth": int(((b[:, 3] > 0) & (a[:, 3] < 0)).sum())}


# UAV.state_PathPlan's 80 probes (UAV.py:533-555,562-566) as the kernel takes them (env_block.cuh probe_offset): 3 planar 5 x 5
# grids at 1 / 5 / 10 m for slots 11..85, then 1..5 m below for slots 90..94
_G = np.array([1, 5, 10]).repeat(25)
_IJ = np.tile(np.arange(25), 3)
PROBE_DX = np.r_[_G * (_IJ // 5 - 2), np.zeros(5, np.int64)].astype(np.float64)
PROBE_DY = np.r_[_G * (_IJ % 5 - 2), np.zeros(5, np.int64)].astype(np.float64)
PROBE_SLOT = np.r_[11:86, 90:95]


def probe_points(px, py, pz):
    """[n, 80, 3] probe points of n UAVs in observation-slot order PROBE_SLOT, each coordinate the IEEE operation the kernel
    performs: px + dx, py + dy at z = pz for the planar probes, px, py at pz - (k + 1) for the probes below."""
    px, py, pz = (np.asarray(v, np.float64).reshape(-1, 1) for v in (px, py, pz))
    x = np.concatenate([px + PROBE_DX[None, :75], np.repeat(px, 5, 1)], 1)
    y = np.concatenate([py + PROBE_DY[None, :75], np.repeat(py, 5, 1)], 1)
    z = np.concatenate([np.repeat(pz, 75, 1), pz - np.arange(1.0, 6.0)[None]], 1)
    return np.stack([x, y, z], 2)


def obstacle_run(tab, length, width):
    """One run() of every row (x, y, vx, vy) of tab, in place, each IEEE operation in the rule's order."""
    for r in tab:
        x, y, vx, vy = (float(v) for v in r)
        x = x + vx
        if x < 0:
            x, vx = -x, -vx
        elif x > length:
            x, vx = length - (x - length), -vx
        y = y + vy
        if y < 0:
            y, vy = -y, -vy
        elif y > width:
            y, vy = width - (y - width), -vy
        r[:] = (x, y, vx, vy)


class MovingCity:
    """An OracleCity whose centres follow tab [n, 4]; with apf, the oracle's APF velocities follow its signs."""

    def __init__(self, length, width, h, buildings, tab, vz=None, apf=False):
        self.city = O.OracleCity(length, width, h, np.array(buildings, np.float64))     # its own copy: the caller's stays put
        self.len, self.width = float(length), float(width)
        self.tab = np.array(tab, np.float64).reshape(-1, 4)
        self.apf = apf
        if apf:
            v = np.zeros((self.tab.shape[0], 3))
            v[:, 2] = 0.0 if vz is None else vz
            O.set_apf(v)
        self.sync()

    def sync(self):
        self.city.buildings[:, 0] = self.tab[:, 0]
        self.city.buildings[:, 1] = self.tab[:, 1]
        if self.apf:
            O._apf_keep[:, 0] = self.tab[:, 2]
            O._apf_keep[:, 1] = self.tab[:, 3]

    def advance(self):
        obstacle_run(self.tab, self.len, self.width)
        self.sync()

    def close(self):
        if self.apf:
            O.set_apf(None)


def step(mc, batch, actions, mode):
    """One step of batch on O_t, then the table's run(); returns (reward, done, info, coll, obs on O_{t+1})."""
    rew, done, info, coll, _ = batch.step_(actions, mode, want_obs=False)
    mc.advance()
    return rew, done, info, coll, batch.state()
