"""A Python restatement of the control-latency draw (deepmimic_b200/csrc/kernels/dm_latency.cuh: lat_draw) for the CPU shim test and the GPU
tests: the delay of an environment's episode with reset counter r is lo + min(hi - lo, floor(u (hi - lo + 1))), u the library's uniform."""
import math

from tests.push_schedule_ref import u01

LAT_SEED_KEY = 0x6c6174656e6379   # "latency"


def lat_seed(handle_seed):
    return handle_seed ^ LAT_SEED_KEY


def draw(lo, hi, seed, env, resets):
    """the delay in updates; seed is the stream's"""
    span = hi - lo
    return lo + min(span, int(math.floor(u01(seed, env, resets) * float(span + 1))))
