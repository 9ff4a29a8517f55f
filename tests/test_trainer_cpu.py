"""The training iteration's rules of deepmimic_b200/trainer.py against numpy restatements: the device replay storage (ReplayBufferRandStorage),
TarClipFrac stepsize control, the discriminator's step count, the exploration lerp and RLAgent._train's InitSamples / NormalizerSamples phases."""
import math

import numpy as np
import pytest

from deepmimic_b200 import trainer as tr


def _rows(n, start, width=3):
    import torch
    return torch.arange(start, start + n, dtype=torch.float32)[:, None].repeat(1, width)


def test_replay_fills_in_order_then_overwrites_distinct_slots():
    import torch
    buf = tr.DeviceReplayBuffer(10, 3, "cpu", seed=4)
    buf.store(_rows(3, 100)); buf.store(_rows(4, 200))
    assert buf.size == 7 and buf.total_count == 7
    np.testing.assert_array_equal(buf.filled()[:, 0].numpy(), [100, 101, 102, 200, 201, 202, 203])
    # a store that crosses the end: 3 rows take the free slots in order, the other 2 overwrite distinct uniformly drawn slots
    g = torch.Generator(); g.set_state(buf.generator.get_state())
    want = buf.rows.clone()
    want[7:10] = _rows(3, 300)
    want[torch.randperm(10, generator=g)[:2]] = _rows(2, 303)
    buf.store(_rows(5, 300))
    assert buf.size == 10 and buf.total_count == 12
    assert torch.equal(buf.rows, want)
    for k in range(20):   # once full, a store of n rows replaces exactly n distinct slots
        before = buf.rows.clone()
        new = _rows(6, 1000 + 10 * k)
        buf.store(new)
        changed = (buf.rows != before).any(dim=1)
        assert int(changed.sum()) == 6
        assert sorted(buf.rows[changed, 0].tolist()) == new[:, 0].tolist()
    assert buf.size == 10


def test_replay_samples_only_filled_slots_and_refuses_long_stores():
    buf = tr.DeviceReplayBuffer(50, 2, "cpu", seed=1)
    buf.store(_rows(3, 7, width=2))
    s = buf.sample(2000)
    assert tuple(s.shape) == (2000, 2) and set(s[:, 0].tolist()) == {7.0, 8.0, 9.0}
    with pytest.raises(ValueError, match="smaller than the buffer"):
        buf.store(_rows(50, 0, width=2))
    with pytest.raises(ValueError, match="empty"):
        tr.DeviceReplayBuffer(5, 2, "cpu").sample(1)


def test_replay_is_bit_identical_under_the_same_seed_and_round_trips():
    import torch
    a, b, c = (tr.DeviceReplayBuffer(16, 4, "cpu", seed=s) for s in (9, 9, 10))
    for k in range(6):
        x = torch.randn(7, 4, generator=torch.Generator().manual_seed(k))
        for buf in (a, b, c):
            buf.store(x)
    assert torch.equal(a.rows, b.rows) and torch.equal(a.sample(33), b.sample(33))
    assert not torch.equal(a.rows, c.rows)
    d = tr.DeviceReplayBuffer(16, 4, "cpu", seed=0)
    d.load_state_dict(a.state_dict())
    assert d.size == a.size and d.total_count == a.total_count and torch.equal(d.rows, a.rows)
    assert torch.equal(d.sample(5), a.sample(5))


def _np_stepsize(s, cf, tar, decay, it):
    if tar >= 0 and it > 5:
        if cf > 1.5 * tar:
            s = s * decay
        elif cf < tar / 1.5:
            s = s / decay
        s = float(np.clip(s, 1e-8, 1e-2))
    return s


@pytest.mark.parametrize("it", [0, 5, 6, 40])
@pytest.mark.parametrize("cf", [0.0, 0.1, 0.2 / 1.5 - 1e-6, 0.2 / 1.5, 0.2, 0.3, 0.3 + 1e-6, 0.9])
def test_actor_stepsize_control(it, cf):
    for s, tar, decay in ((2.5e-6, 0.2, 0.5), (9e-3, 0.2, 0.5), (1.5e-8, 0.2, 2.0), (1e-5, -1.0, 0.5)):
        assert tr.update_actor_stepsize(s, cf, tar, decay, it) == _np_stepsize(s, cf, tar, decay, it)
    assert tr.update_actor_stepsize(2.5e-6, 0.9, 0.2, 0.5, 5) == 2.5e-6               # the warm-up
    assert tr.update_actor_stepsize(9e-3, 0.0, 0.2, 0.5, 6) == 1e-2                   # clipped above
    assert tr.update_actor_stepsize(1.5e-8, 0.9, 0.2, 0.5, 6) == 1e-8                 # clipped below


def test_disc_steps_per_iter():
    for samples, spb, bs in ((32 * 4096, 1, 256), (1000, 2, 256), (255, 1, 256), (4096, 3, 4096)):
        assert tr.disc_steps_per_iter(samples, spb, bs) == int(np.ceil(spb * samples / bs))
    assert tr.disc_steps_per_iter(1000, 2, 256) == 8


def test_exploration_lerp():
    beg = dict(Rate=1.0, InitActionRate=1.0, Noise=0.05, NoiseInternal=0.0, Temp=20.0)
    end = dict(Rate=0.2, InitActionRate=0.01, Noise=0.05, NoiseInternal=0.0, Temp=0.001)
    for samples, anneal in ((0, 64e6), (16e6, 64e6), (64e6, 64e6), (1e9, 64e6), (5, 0)):
        t = float(np.clip(samples / anneal, 0.0, 1.0)) if anneal > 0 else 0.0
        got = tr.exploration_params(beg, end, samples, anneal)
        for k in tr.EXP_PARAM_KEYS:
            assert math.isclose(got[k], (1 - t) * beg[k] + t * end[k], rel_tol=0, abs_tol=1e-12)
    assert tr.exploration_params(beg, end, 32e6, 64e6)["Rate"] == pytest.approx(0.6)


def test_train_schedule_init_and_normalizer_phases():
    """windows of 1000 samples, InitSamples 2500, NormalizerSamples 4200: windows 1-2 only record and update the normalisers, window 3 crosses
    InitSamples (initialises, no training), windows 4-5 train and still update the normalisers (the fifth crosses NormalizerSamples and is the
    last one recorded), from window 6 on only training"""
    initialized, need = False, True
    seen = []
    for w in range(1, 9):
        train, initialized, update, need = tr.train_schedule(1000 * w, initialized, need, 2500, 4200)
        seen.append((train, update))
    assert seen == [(False, True), (False, True), (False, True), (True, True), (True, True), (True, False), (True, False), (True, False)]
