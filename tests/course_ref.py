"""A numpy restatement of the goal courses (deepmimic_b200/csrc/kernels/dm_course.cuh) for the CPU shim test and the GPU tests: the heading
course's goal at an episode time, the target course's waypoint advance, and the record of a course call."""
import math

import numpy as np

GOAL_POINT_DIST = 1.5   # m: the heading record's goal point ahead of the root


def heading_goal(rows, tau):
    """(h, v) of the heading course rows [n, 3] (t, h, v) at episode time tau: row 0 before t_0, the last row from t_{n-1} on, linear between"""
    rows = np.asarray(rows, dtype=np.float64)
    if tau < rows[0, 0]:
        return float(rows[0, 1]), float(rows[0, 2])
    if tau >= rows[-1, 0]:
        return float(rows[-1, 1]), float(rows[-1, 2])
    k = int(np.searchsorted(rows[:, 0], tau, side="right")) - 1   # t_k <= tau < t_{k+1}
    w = (tau - rows[k, 0]) / (rows[k + 1, 0] - rows[k, 0])
    lerp = lambda a, b: a + (b - a) * w
    return float(lerp(rows[k, 1], rows[k + 1, 1])), float(lerp(rows[k, 2], rows[k + 1, 2]))


class Course:
    """one environment's course and progress; kind "heading" (rows (t, h, v)) or "target" (rows (dx, dz[, unused])).  goal is the task
    block's goal: (h, v) or the waypoint (x, z)"""

    def __init__(self, kind, rows, succ_dist=0.5):
        self.kind, self.rows, self.succ_dist = kind, np.asarray(rows, dtype=np.float64), succ_dist

    def waypoint(self):
        k = min(self.active, len(self.rows) - 1)
        return self.org[0] + self.rows[k, 0], self.org[1] + self.rows[k, 1]

    def _write_goal(self, tau):
        self.goal = heading_goal(self.rows, tau) if self.kind == "heading" else self.waypoint()

    def record(self, rx, rz, tau):
        if self.kind == "heading":
            h, v = self.goal
            ch, sh = math.cos(h), math.sin(h)
            dt = tau - self.prev[2]
            along = cross = 0.0
            if dt > 0:
                dx, dz = rx - self.prev[0], rz - self.prev[1]
                along = (ch * dx - sh * dz) / dt - v
                cross = (-sh * dx - ch * dz) / dt
            return np.array([rx + GOAL_POINT_DIST * ch, rz - GOAL_POINT_DIST * sh, along, cross])
        wx, wz = self.waypoint()
        return np.array([wx, wz, float(self.active), math.hypot(rx - wx, rz - wz)])

    def start(self, rx, rz, tau):
        """a reset or the setter: origin and previous root here, goal for tau; returns the record of no interval"""
        self.active, self.org, self.prev = 0, (rx, rz), (rx, rz, tau)
        self._write_goal(tau)
        return self.record(rx, rz, tau)

    def advance(self, rx, rz):
        while self.active < len(self.rows):
            wx, wz = self.org[0] + self.rows[self.active, 0], self.org[1] + self.rows[self.active, 1]
            if not (rx - wx) ** 2 + (rz - wz) ** 2 < self.succ_dist ** 2:
                break
            self.active += 1

    def step(self, rx, rz, tau):
        """after a step launch that ended at root (rx, rz) and episode time tau: the record (after the advance in the target scene), then the
        goal for tau"""
        if self.kind == "target":
            self.advance(rx, rz)
        rec = self.record(rx, rz, tau)
        self.prev = (rx, rz, tau)
        self._write_goal(tau)
        return rec
