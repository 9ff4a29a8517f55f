"""Control latency on the CPU: the shared host / device delay draw of dm_latency.cuh through a g++ shim against the Python restatement
(tests/latency_ref.py), bit for bit, with its spread over [lo, hi]; the seconds-to-updates rounding of the Python layer; the train and run
options; the Trainer's run record; and the ptxas resources of the latency step kernels against the dynamics kernels'."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import latency_ref as ref
from tests.native import nvcc, ptxas_report, shared_library

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def shim():
    L = shared_library(os.path.join(HERE, "latency_shim.cpp"), ["-O2"])
    L.shim_lat_draw.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int]
    L.shim_lat_seed_key.restype = C.c_uint64
    return L


@pytest.mark.parametrize("lo,hi", [(0, 19), (3, 7), (0, 1), (19, 19), (5, 5), (0, 0)])
@pytest.mark.parametrize("handle_seed", [0, 21])
def test_shim_matches_the_restatement(shim, lo, hi, handle_seed):
    """2000 (global env id, reset counter) pairs, ids up to 2^40: the shim's delay equals the restatement's; lo = hi always gives lo"""
    assert shim.shim_lat_seed_key() == ref.LAT_SEED_KEY and shim.shim_lat_bytes() == 528
    seed = ref.lat_seed(handle_seed)
    rng = np.random.default_rng(lo * 100 + hi + handle_seed)
    envs = list(range(1000)) + [int(x) for x in rng.integers(0, 1 << 40, size=1000)]
    for e in envs:
        r = int(rng.integers(0, 1 << 20))
        got = shim.shim_lat_draw(lo, hi, seed, e, r)
        assert got == ref.draw(lo, hi, seed, e, r), (e, r)
        assert lo <= got <= hi
        if lo == hi:
            assert got == lo


@pytest.mark.parametrize("lo,hi", [(0, 19), (4, 11)])
def test_draws_cover_the_range_uniformly(shim, lo, hi):
    """20000 draws over environments and episodes reach every integer of [lo, hi], and a chi-square test against the uniform passes"""
    from scipy.stats import chisquare
    seed = ref.lat_seed(5)
    d = np.array([shim.shim_lat_draw(lo, hi, seed, e, r) for e in range(200) for r in range(100)])
    counts = np.bincount(d - lo, minlength=hi - lo + 1)
    assert counts.size == hi - lo + 1 and np.all(counts > 0)
    assert chisquare(counts).pvalue > 1e-3


def test_seconds_round_to_updates_and_refuse():
    from deepmimic_b200.capi import UPDATE_DT, latency_updates
    assert latency_updates(0.0, 20) == 0 and latency_updates(0.0167, 20) == 10 and latency_updates(0.0317, 20) == 19
    assert latency_updates(19.4 * UPDATE_DT, 20) == 19 and latency_updates(0.4 * UPDATE_DT, 20) == 0
    for bad in (19.6 * UPDATE_DT, -0.6 * UPDATE_DT, 0.05, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            latency_updates(bad, 20)


def test_python_limit_is_the_library_limit():
    """the Python layer's updates per action (the option checks' limit) is the library's kUpdatesPerAction"""
    import re
    from deepmimic_b200.capi import UPDATES_PER_ACTION
    from tests.native import CSRC
    src = open(os.path.join(CSRC, "capi.cu")).read()
    assert int(re.search(r"constexpr int kUpdatesPerAction = (\d+);", src).group(1)) == UPDATES_PER_ACTION


def test_train_option_parses_and_refuses():
    from deepmimic_b200.train import build_parser
    ap = build_parser()
    assert ap.parse_known_args([])[0].rand_latency is None
    assert ap.parse_known_args(["--rand_latency", "0,0.03"])[0].rand_latency == [0.0, 0.03]
    for bad in ("0.03,0", "0,0.05", "-0.01,0.01", "a,b", "0.01", "nan,0.01", "0,inf"):
        with pytest.raises(SystemExit):
            ap.parse_known_args(["--rand_latency", bad])


def test_run_option_parses_and_refuses():
    from deepmimic_b200.capi import UPDATE_DT
    from deepmimic_b200.run import build_parser
    ap = build_parser()
    assert ap.parse_known_args([])[0].latency_sweep is None
    got = ap.parse_known_args(["--latency_sweep", "0,0.0167,0.0317"])[0].latency_sweep
    assert got == [0.0, 10 * UPDATE_DT, 19 * UPDATE_DT]
    for bad in ("", "a", "0,0.04", "-0.01", "nan", "0,inf"):
        with pytest.raises(SystemExit):
            ap.parse_known_args(["--latency_sweep", bad])


def test_trainer_record_and_checkpoint_refusal():
    """the run record carries the bounds rounded to whole updates, only when given; load_state_dict refuses a checkpoint of other bounds or
    none, before anything else is read"""
    from deepmimic_b200.capi import UPDATE_DT
    from deepmimic_b200.trainer import Trainer, latency_record
    assert latency_record(None) is None
    assert latency_record((0.0, 0.03)) == [0.0, 18 * UPDATE_DT]
    for bad in ((0.03, 0.0), (0.0, 0.05), (0.01,), (float("nan"), 0.01)):
        with pytest.raises(ValueError):
            latency_record(bad)
    t = Trainer.__new__(Trainer)
    t.torch, t.ro = None, None
    t.run = dict(model_files=None, latency_randomization=latency_record((0.0, 0.03)))
    with pytest.raises(ValueError, match="latency randomisation"):
        t.load_state_dict(dict(run=dict(model_files=None)))
    with pytest.raises(ValueError, match="latency randomisation"):
        t.load_state_dict(dict(run=dict(model_files=None, latency_randomization=latency_record((0.0, 0.02)))))


@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
def test_latency_step_kernel_resources(tmp_path):
    """ptxas's figures for the four latency step kernels: registers, stack frame and spills no worse than the matching dynamics kernel's"""
    rep = ptxas_report(os.path.join("kernels", "dm_step.cu"), str(tmp_path))
    for w in (16, 32):
        for task in (0, 1):
            (lat,) = [e for e in rep if "dm_step_latency_kernelILi%dELb%dE" % (w, task) in e]
            (dyn,) = [e for e in rep if "dm_step_dyn_kernelILi%dELb%dE" % (w, task) in e]
            (lregs, lfuncs), (dregs, dfuncs) = rep[lat], rep[dyn]
            assert lregs <= dregs, (w, task, lregs, dregs)
            assert all(a <= b for a, b in zip(lfuncs[0][1:], dfuncs[0][1:])), (w, task, lfuncs[0], dfuncs[0])
