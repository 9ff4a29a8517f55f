"""A Python restatement of the push schedule (deepmimic_b200/csrc/kernels/dm_push.cuh: push_schedule_env) and of its draw stream, for the
CPU shim test and the GPU tests.  Plain IEEE double arithmetic with one rounding per operation (no fused multiply-add), glibc's sin / cos
through math, and float32 rounding of the force as the push table stores it."""
import math

import numpy as np

PUSH_SEED_KEY = 0x707573686573   # "pushes"
_M = (1 << 64) - 1


def u01(seed, a, b):
    """the library's counter-based uniform (dm_task.cuh: task_u01, splitmix64's finaliser)"""
    z = (seed + 0x9E3779B97F4A7C15 * ((a * 2654435761 + b + 1) & _M)) & _M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M
    z ^= z >> 31
    return float(z >> 11) * (1.0 / 9007199254740992.0)


def push_seed(handle_seed):
    return handle_seed ^ PUSH_SEED_KEY


def _lerp(lohi, u):
    return lohi[0] + u * (lohi[1] - lohi[0])


class Entry:
    """one push-table entry: body (-1 none), force (3 float32), start, duration"""

    def __init__(self, body=-1, force=(0.0, 0.0, 0.0), start=0.0, duration=0.0):
        self.body, self.force, self.start, self.duration = int(body), np.asarray(force, dtype=np.float32).copy(), float(start), float(duration)


def schedule_env(bodies, force, duration, gap, seed, env, resets, timer, block, entry):
    """one environment's schedule step.  block: [reset counter seen, draw counter k, last_end] (a list, updated); entry: Entry (updated).
    seed is the stream's seed (push_seed of the handle's), env the global environment id."""
    if float(resets) != block[0]:
        block[0], block[1], block[2] = float(resets), 0.0, 0.0
    if entry.body != -1:
        return
    k = int(block[1])
    u = [u01(seed, env, k + i) for i in range(5)]   # gap, body index, magnitude, direction angle, duration
    g = _lerp(gap, u[0])
    i = min(int(u[1] * float(len(bodies))), len(bodies) - 1)
    mag = _lerp(force, u[2])
    ang = (2.0 * math.pi) * u[3]
    dur = _lerp(duration, u[4])
    block[1] = float(k + 5)
    start = max(block[2] + g, timer)
    entry.body = int(bodies[i])
    entry.force = np.array([mag * math.cos(ang), 0.0, mag * math.sin(ang)], dtype=np.float32)
    entry.start, entry.duration = start, dur
    block[2] = start + dur
