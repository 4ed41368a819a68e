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
        self.city = O.OracleCity(length, width, h, buildings)
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
