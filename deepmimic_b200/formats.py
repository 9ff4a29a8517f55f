"""On-disk formats of the reference next to the hot path (SURVEY.md section 8f, rank 4): written from scratch so that files produced here load in
the reference and files produced by the reference load here.  Pure host code, no device work.

  motion clip    cMotion::Output / LoadJson           R/DeepMimicCore/anim/Motion.cpp:104-141,303-360,581-646
  state snapshot cCharacter::WriteState / ReadState   R/DeepMimicCore/anim/Character.cpp:320-385,434-443
  training log   Logger.log_tabular / dump_tabular    R/util/logger.py:63-127 (fixed-width 25-character columns)
  animated PNG   the APNG extension of PNG (acTL / fcTL / fdAT chunks): rendered episodes and motion files (deepmimic_b200/render.py)

The BVH importer (R/DeepMimicCore/util/BVHReader.cpp) is deepmimic_b200/bvh.py."""
import binascii
import json
import re
import struct
import zlib
from fractions import Fraction

import numpy as np


def _vec(values):
    """cJsonUtil::BuildVectorJson (util/JsonUtil.cpp:39-60): "%20.10f" entries separated by commas."""
    return "[" + ",".join("%20.10f" % float(v) for v in values) + "]"


def write_motion(path, frames, durations, loop="wrap", cycle_sync_root_pos=False, cycle_sync_root_rot=False, cycle_sync_root_height=False):
    """frames: [F, D] poses (root position 3, root quaternion w x y z, joints); durations: F frame durations (the last one is written as 0,
    like the reference does).  Layout of cMotion::Output."""
    frames = np.asarray(frames, dtype=np.float64)
    durations = np.asarray(durations, dtype=np.float64)
    if frames.ndim != 2 or len(durations) != frames.shape[0]:
        raise ValueError("frames must be [F, D] with one duration per frame")
    if loop not in ("none", "wrap"):
        raise ValueError("Unsupported loop mode: %s" % loop)
    b = lambda v: "true" if v else "false"
    with open(path, "w") as f:
        f.write("{\n\"Loop\": \"%s\",\n" % loop)
        f.write("\"CycleSyncRootPos\": %s,\n\"CycleSyncRootRot\": %s,\n\"CycleSyncRootHeight\": %s,\n\n" % (b(cycle_sync_root_pos), b(cycle_sync_root_rot), b(cycle_sync_root_height)))
        f.write("\"Frames\":\n[\n")
        n = frames.shape[0]
        rows = []
        for i in range(n):
            dur = durations[i] if i < n - 1 else 0.0
            rows.append(_vec(np.concatenate([[dur], frames[i]])))
        f.write(",\n".join(rows))
        f.write("\n]\n}")


def read_motion(path):
    """Returns dict(loop, frames [F, D], durations [F], flags): the raw file content (no recentring, no quaternion normalisation -- the
    loaders of the simulation do that, csrc/host/assets.hpp)."""
    root = json.load(open(path))
    fr = np.asarray(root["Frames"], dtype=np.float64)
    if fr.ndim != 2 or fr.shape[0] == 0:
        raise ValueError("Failed to load motion from file %s" % path)
    return dict(loop=root.get("Loop", "none"), frames=fr[:, 1:].copy(), durations=fr[:, 0].copy(),
                cycle_sync_root_pos=bool(root.get("CycleSyncRootPos", False)), cycle_sync_root_rot=bool(root.get("CycleSyncRootRot", False)),
                cycle_sync_root_height=bool(root.get("CycleSyncRootHeight", False)))


def write_state(path, pose, vel):
    """cCharacter::BuildStateJson: {"Pose": [...], "Vel": [...]} with the reference's number format."""
    with open(path, "w") as f:
        f.write("{\n\"Pose\":" + _vec(pose) + ",\n\"Vel\":" + _vec(vel) + "\n}")


def read_state(path):
    root = json.load(open(path))
    return (np.asarray(root["Pose"], dtype=np.float64) if "Pose" in root else None, np.asarray(root["Vel"], dtype=np.float64) if "Vel" in root else None)


class TableLog:
    """The learner's tabular log (R/util/logger.py): the first row fixes the headers; every cell is left-aligned in 25 characters; floats print
    through str().  append=True continues an existing log (a resumed run): its header line fixes the headers and is not written again."""

    def __init__(self, path, append=False):
        import os
        self.headers, self.row, self.first = [], {}, True
        if append and os.path.exists(path) and os.path.getsize(path) > 0:
            with open(path) as f:
                self.headers = f.readline().split()
            self.first = False
        self.file = open(path, "a" if append else "w")

    def log_tabular(self, key, val):
        if self.first and key not in self.headers:
            self.headers.append(key)
        elif key not in self.headers:
            raise KeyError("Trying to introduce a new key %s that you didn't include in the first iteration" % key)
        self.row[key] = val

    def dump_tabular(self):
        template = "{:<25}" * len(self.headers)
        if self.first:
            self.file.write(template.format(*self.headers) + "\n")
        self.file.write(template.format(*map(str, (self.row.get(k, "") for k in self.headers))) + "\n")
        self.file.flush()
        self.row.clear()
        self.first = False

    def close(self):
        self.file.close()


def read_table_log(path):
    """Reads a log written by the reference's Logger (or TableLog): dict of header -> float array (NaN for empty cells)."""
    lines = [l.rstrip("\n") for l in open(path) if l.strip()]
    if not lines:
        return {}
    headers = re.split(r"\s+", lines[0].strip())
    cols = {h: [] for h in headers}
    for l in lines[1:]:
        cells = re.split(r"\s+", l.strip())
        for h, c in zip(headers, cells + [""] * (len(headers) - len(cells))):
            try:
                cols[h].append(float(c))
            except ValueError:
                cols[h].append(float("nan"))
    return {h: np.asarray(v) for h, v in cols.items()}


def _png_chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", binascii.crc32(kind + data) & 0xFFFFFFFF)


def write_apng(path, frames, durations):
    """An animated PNG of T RGB frames: frames is a uint8 array [T, H, W, 3] or an iterable of T [H, W, 3] arrays (consumed one frame at a
    time), durations the T frame delays in seconds.  Frame 0 is also the default image (IDAT), so a viewer without APNG support shows it;
    every frame has its own fcTL delay, the nearest fraction with a 16-bit denominator; the animation loops.  Pixels are stored losslessly."""
    durations = [float(d) for d in durations]
    if not durations or any(not (d >= 0.0) or d == float("inf") for d in durations):
        raise ValueError("write_apng: need one finite duration >= 0 per frame")
    with open(path, "wb") as f:
        n, shape = 0, None
        for frame in frames:
            frame = np.asarray(frame)
            if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3 or (shape is not None and frame.shape != shape):
                raise ValueError("write_apng: every frame must be uint8 [H, W, 3] of one size, got %s %s" % (frame.dtype, frame.shape))
            if n >= len(durations):
                raise ValueError("write_apng: more frames than durations")
            H, W = frame.shape[:2]
            if n == 0:
                shape = frame.shape
                f.write(b"\x89PNG\r\n\x1a\n")
                f.write(_png_chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)))
                f.write(_png_chunk(b"acTL", struct.pack(">II", len(durations), 0)))
            delay = Fraction(durations[n]).limit_denominator(65535)
            if delay.numerator > 65535:
                raise ValueError("write_apng: a frame duration of %g s does not fit a 16-bit delay" % durations[n])
            seq = 0 if n == 0 else 2 * n - 1   # fcTL and fdAT chunks share one sequence: fcTL 0, (fcTL 1, fdAT 2), (fcTL 3, fdAT 4), ...
            f.write(_png_chunk(b"fcTL", struct.pack(">IIIIIHHBB", seq, W, H, 0, 0, delay.numerator, delay.denominator, 0, 0)))
            rows = np.concatenate([np.zeros((H, 1), dtype=np.uint8), frame.reshape(H, 3 * W)], axis=1)   # filter type 0 on every row
            data = zlib.compress(rows.tobytes(), 6)
            f.write(_png_chunk(b"IDAT", data) if n == 0 else _png_chunk(b"fdAT", struct.pack(">I", seq + 1) + data))
            n += 1
        if n != len(durations):
            raise ValueError("write_apng: %d frames for %d durations" % (n, len(durations)))
        f.write(_png_chunk(b"IEND", b""))
