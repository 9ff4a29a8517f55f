"""Per-environment dynamics on the CPU: the shared host / device draw of dm_dynamics.cuh through a g++ shim against the Python restatement
(tests/dynamics_ref.py), bit for bit, over many environments and reset counters, with lumped leaves copying their parent's factor; the
environment's argument checks; and the ptxas resources of the dynamics step kernels."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests import dynamics_ref as ref
from tests.test_step_resources_cpu import nvcc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """dm_dynamics.cuh compiled with g++ (no contraction of a product into an add, as on the device with its explicit roundings)"""
    so = str(tmp_path_factory.mktemp("dyn_shim") / "libdynamics_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, "dynamics_shim.cpp"),
                           "-o", so])
    L = C.CDLL(so)
    dp, ip, fp = C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_float)
    L.shim_dyn_draw.argtypes = [dp, C.c_uint64, C.c_uint64, C.c_int, C.c_int, ip, fp, fp]
    L.shim_dyn_seed_key.restype = C.c_uint64
    return L


def _shim_draw(L, lohi, seed, env, resets, leaf_parent, masses):
    lh = np.ascontiguousarray(lohi, dtype=np.float64)
    lp = np.ascontiguousarray(leaf_parent, dtype=np.int32)
    ms = np.ascontiguousarray(masses, dtype=np.float32)
    out = np.zeros(L.shim_dyn_floats(), dtype=np.float32)
    L.shim_dyn_draw(lh.ctypes.data_as(C.POINTER(C.c_double)), seed, env, resets, len(lp), lp.ctypes.data_as(C.POINTER(C.c_int)),
                    ms.ctypes.data_as(C.POINTER(C.c_float)), out.ctypes.data_as(C.POINTER(C.c_float)))
    return out


def _char(asset_root, name):
    return os.path.join(asset_root, "data", "characters", name + ".txt")


def test_lumped_leaves_of_the_characters(asset_root):
    """humanoid3d's wrists (links 8 and 14) are lumped into the elbows; dog3d has no lumped leaf"""
    hum = ref.lumped_leaves(_char(asset_root, "humanoid3d"))
    assert {l: p for l, p in enumerate(hum) if p >= 0} == {8: 7, 14: 13}
    assert all(p < 0 for p in ref.lumped_leaves(_char(asset_root, "dog3d")))


BOUNDS = [(0.4, 1.2, 0.8, 1.2, 0.7, 1.3, 0.5, 1.0, 0.7, 1.3),
          (0.0, 2.0, 0.0, 0.0, 1.0, 1.0, 0.0, 3.0, 1e-3, 10.0),     # zero-width and zero-lo ranges
          (1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0)]        # the plain model


@pytest.mark.parametrize("char", ["humanoid3d", "dog3d"])
@pytest.mark.parametrize("k", range(len(BOUNDS)))
def test_shim_matches_the_restatement_bit_for_bit(shim, asset_root, char, k):
    """every factor and the total mass of 300 environments (ids up to 2^40) at reset counters 0 .. 300, shim against restatement, bit for bit;
    a lumped leaf carries its parent's draw; every factor lies in its [lo, hi]; unit bounds give exactly the plain model's total mass"""
    assert shim.shim_dyn_seed_key() == ref.DYN_SEED_KEY and shim.shim_dyn_floats() == 40
    lohi = BOUNDS[k]
    lp = ref.lumped_leaves(_char(asset_root, char))
    ms = ref.link_masses(_char(asset_root, char))
    nl = len(lp)
    seed = ref.dyn_seed(77 + k)
    rng = np.random.default_rng(k)
    envs = list(range(100)) + [int(x) for x in rng.integers(0, 1 << 40, size=200)]
    for e in envs:
        r = int(rng.integers(0, 300))
        got = _shim_draw(shim, lohi, seed, e, r, lp, ms)
        want = ref.draw_env(lohi, seed, e, r, lp)
        assert got[:4 + nl].tobytes() == want.tobytes(), (e, r)
        assert np.all(got[4 + nl:36] == 1.0) and np.all(got[37:] == 0.0)
        assert got[36] == ref.total_mass(ms, want)
        for j in range(5):
            sel = want[j:j + 1] if j < 4 else want[4:]
            assert np.all(sel >= np.float32(lohi[2 * j])) and np.all(sel <= np.float32(lohi[2 * j + 1]))
        for l, p in enumerate(lp):
            if p >= 0:
                assert want[4 + l] == want[4 + p]
    if k == 2:
        assert ref.total_mass(ms, np.ones(4 + nl, dtype=np.float32)) == np.float32(sum(ms))


def test_draws_differ_between_episodes_and_environments(shim, asset_root):
    """the stream moves with the reset counter and the global id: 50 episodes x 50 environments draw 2500 frictions, equal only where two
    draws round to one float32 (a few in 2500 at this width)"""
    lp = ref.lumped_leaves(_char(asset_root, "humanoid3d"))
    seed = ref.dyn_seed(5)
    fr = {float(ref.draw_env(BOUNDS[0], seed, e, r, lp)[0]) for e in range(50) for r in range(50)}
    assert len(fr) >= 2490


def test_env_argument_checks():
    """DeepMimicBatchEnv.set_dynamics / set_dynamics_randomization refuse wrong shapes before the library sees them"""
    from deepmimic_b200.env import DeepMimicBatchEnv

    class Dims:
        num_joints = 15

    class Core:
        num_envs, dims = 4, Dims()

        def set_dynamics(self, f):
            self.f = f

        def set_dynamics_randomization(self, lohi):
            self.lohi = lohi
    env = DeepMimicBatchEnv.__new__(DeepMimicBatchEnv)
    env._core = Core()
    env._pre = lambda: None
    with pytest.raises(ValueError, match="friction must have shape"):
        env.set_dynamics(friction=np.ones(3))
    with pytest.raises(ValueError, match="mass must have shape"):
        env.set_dynamics(mass=np.ones((4, 14)))
    with pytest.raises(ValueError, match="kd must be a"):
        env.set_dynamics_randomization(kd=(1.0, 2.0, 3.0))
    env.set_dynamics(kp=np.full(4, 2.0), mass=np.full((4, 15), 1.5))
    f = env._core.f
    assert f.dtype == np.float32 and f.shape == (4, 19)
    assert np.all(f[:, 1] == 2.0) and np.all(f[:, [0, 2, 3]] == 1.0) and np.all(f[:, 4:] == 1.5)
    env.set_dynamics_randomization(friction=(0.5, 1.5), mass=(0.8, 1.2))
    assert env._core.lohi == [0.5, 1.5, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.8, 1.2]


@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
def test_dynamics_step_kernel_resources(tmp_path):
    """ptxas's figures for the four dynamics step kernels, pinned at what they reach: 128 registers each (the launch plan's count); for the
    imitate instantiations no stack beyond the W = 32 kernel's 40 B sin / cos frame (W = 16: 48 B with 12 B of spills around the collision
    pass) and none in their routines.  The task instantiations keep the task code's frame, as the push kernels do."""
    from tests.test_step_resources_cpu import CSRC, makefile_flags
    r = subprocess.run([nvcc()] + makefile_flags() + ["-Xptxas", "-v", "-c", os.path.join("kernels", "dm_step.cu"), "-o", str(tmp_path / "o.o")],
                       cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    want = {(16, 0): (48, 12, 12), (32, 0): (40, 0, 0), (16, 1): (352, 24, 0), (32, 1): (368, 36, 0)}
    for (w, task), (frame, stores, loads) in want.items():
        m = re.search(r"Compiling entry function '(\S*dm_step_dyn_kernelILi%dELb%dE\S*)'(.*?)(?=Compiling entry function|\Z)" % (w, task), r.stdout, re.S)
        assert m, (w, task)
        entry, body = m.group(1), m.group(2)
        funcs = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", body)
        assert funcs[0][0] == entry and tuple(int(x) for x in funcs[0][1:]) == (frame, stores, loads), (w, task, funcs[0])
        regs = re.search(r"Used (\d+) registers", body)
        assert regs and int(regs.group(1)) == 128, (w, task, regs and regs.group(1))
        if not task:   # the imitate routines store nothing to local memory
            for callee, cfr, cst, cld in funcs[1:]:
                assert int(cfr) == 0 and int(cst) == 0, (w, task, callee, cfr, cst)

def test_train_rand_options_parse_and_refuse(capsys):
    """--rand_* options: each optional, any one switches randomisation on, kinds not given stay 1; bad ranges and a mass lo of 0 refused"""
    from deepmimic_b200.train import build_parser, dynamics_randomization
    from deepmimic_b200.trainer import dynamics_record
    ap = build_parser()
    assert dynamics_randomization(ap.parse_known_args([])[0]) is None
    o = ap.parse_known_args(["--rand_mass", "0.8,1.2", "--rand_friction", "0.5,1.5", "--push_force", "1,2"])[0]
    d = dynamics_randomization(o)
    assert d == dict(mass=[0.8, 1.2], friction=[0.5, 1.5])
    assert dynamics_record(d) == dict(friction=[0.5, 1.5], kp=[1.0, 1.0], kd=[1.0, 1.0], torque_limit=[1.0, 1.0], mass=[0.8, 1.2])
    for bad in (["--rand_kp", "1.2,0.8"], ["--rand_kd", "-1,1"], ["--rand_torque_limit", "1"], ["--rand_friction", "nan,1"]):
        with pytest.raises(SystemExit):
            ap.parse_known_args(bad)
    with pytest.raises(SystemExit, match="--rand_mass needs LO > 0"):
        dynamics_randomization(ap.parse_known_args(["--rand_mass", "0,1"])[0])
    with pytest.raises(ValueError, match="keys among"):
        dynamics_record(dict(gravity=(1, 2)))
    with pytest.raises(ValueError, match="kp must be a"):
        dynamics_record(dict(kp=(1, 2, 3)))


def test_run_dynamics_sweep_option_parses_and_refuses():
    from deepmimic_b200.run import build_parser, dynamics_plan
    ap = build_parser()
    o = ap.parse_known_args(["--dynamics_sweep", "friction=1,0.2"])[0]
    assert o.dynamics_sweep == ("friction", [1.0, 0.2])
    assert list(dynamics_plan(o.dynamics_sweep, 5)) == [1.0, np.float32(0.2), 1.0, np.float32(0.2), 1.0]
    assert ap.parse_known_args([])[0].dynamics_sweep is None
    for bad in ("gravity=1,2", "friction=", "friction=a", "kp=-1", "mass=0,1", "kd=inf"):
        with pytest.raises(SystemExit):
            ap.parse_known_args(["--dynamics_sweep", bad])


def test_trainer_record_and_checkpoint_refusal():
    """the run record carries the randomisation only when given (runs without it keep their record), and load_state_dict refuses a checkpoint
    of another randomisation before anything else is read"""
    from deepmimic_b200.trainer import Trainer
    t = Trainer.__new__(Trainer)
    t.torch, t.ro = None, None
    t.run = dict(model_files=None, dynamics_randomization=dict(friction=[0.5, 1.5], kp=[1.0, 1.0], kd=[1.0, 1.0], torque_limit=[1.0, 1.0],
                                                                mass=[0.8, 1.2]))
    with pytest.raises(ValueError, match="dynamics randomisation"):
        t.load_state_dict(dict(run=dict(model_files=None)))
