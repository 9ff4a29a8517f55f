"""The constructed collision states (tests/contact_states.py) reach, in the CPU oracle, the branch of the link-plane collision pass each
was built for, and a float64 numpy restatement of that pass agrees with the oracle on every state.  Every decision the pass makes on a
state has a margin of at least 10 % of its threshold, so that a kernel evaluating the same formulas in another fp32 order must take the
same branch; the second sub-step's taps do not move under fp32-rounding noise.  Without these checks the library could decay into states
that exercise nothing, or into states on a knife's edge.  Branches no state of a character can reach are listed in UNREACHABLE."""
import numpy as np
import pytest

from tests import contact_states as CS
from tests.oracle_binding import Oracle
from tests.parity_util import SnapLayout
from tools.qd_envelope import perturb

# Nothing is unreachable with the links of contact_states.LINKS.  (The dog's hands would be: their threshold, 0.0041, leaves no usable
# band above the contact-fall tolerance 0.004, so the tolerance states use the head and a finger.)
UNREACHABLE = set()

_LIBS = {}


def _lib(asset_root, ch):
    if ch not in _LIBS:
        _LIBS[ch] = CS.build(Oracle(CS.CHARS[ch]["args"], asset_root), asset_root, ch)
    return _LIBS[ch]


def _mani(lay, snap, j):
    return snap[lay.mani + 48 * j: lay.mani + 48 * j + 48].reshape(4, 12)


def branches(st):
    """the branch names one state's sub-step 1 tap stands for"""
    e = st.expect
    names = ["%s: %s" % (st.cls, CS.EVENTS[e[CS.EVENT]])]
    if e[CS.EVENT] == CS.FULL:
        names.append("full %s: deepest %s replaced %d" % (st.name.split()[0], "new" if e[CS.DEEPEST] < 0 else e[CS.DEEPEST], e[CS.SLOT]))
    if st.cls == "removal":
        names.append("removal mask %04s/%04s" % (format(e[CS.RM_DIST], "b"), format(e[CS.RM_DRIFT], "b")))
    return names


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_every_state_reaches_its_branch_in_the_oracle(asset_root, ch):
    lib = _lib(asset_root, ch)
    orc = Oracle(CS.CHARS[ch]["args"], asset_root)
    wrong, hit = [], {}
    for st in lib:
        taps, _ = CS.contacts(orc, st.snap)
        t1 = tuple(int(x) for x in taps[0, st.link])
        if t1 != st.expect:
            wrong.append("%s: sub-step 1 tap %s, built for %s" % (st, t1, st.expect))
        if st.expect2 is not None and (taps[1, st.link, CS.EVENT], taps[1, st.link, CS.COUNT]) != st.expect2:
            wrong.append("%s: sub-step 2 event / count %s, built for %s" % (st, tuple(taps[1, st.link, [CS.EVENT, CS.COUNT]]), st.expect2))
        others = [j for j in range(orc.num_joints) if j != st.link and (taps[:, j, CS.EVENT] != CS.NONE).any()]
        if others:
            wrong.append("%s: links %s collide too" % (st, others))
        for n in branches(st):
            hit.setdefault(n, []).append(st.name)
    print("%s: %d constructed states" % (ch, len(lib)))
    for n in sorted(hit):
        print("  %-44s %3d states, e.g. %s" % (n, len(hit[n]), hit[n][0]))
    assert not wrong, "\n".join(wrong)
    # the 16 (deepest, replaced) combinations of sortCachedPoints on each of the box, capsule and sphere links
    for what in ("box", "capsule", "sphere"):
        combos = {n for n in hit if n.startswith("full %s:" % what)}
        assert len(combos) == 16, (what, sorted(combos))
    # every non-empty subset of a full cache removed, each with both alternations of distance and drift
    assert len([n for n in hit if n.startswith("removal mask")]) >= 2 * 15
    for cls in ("support", "add", "replace", "full", "refresh", "removal", "fall", "release"):
        assert any(n.startswith(cls + ":") for n in hit), cls


def _margins(dec, thr):
    """decisions closer to their threshold than 10 % of the link's threshold (relative for area leads; >= 1e-3 for a box's down
    direction components and a capsule's end choice)"""
    bad = []
    for kind, v, t in dec:
        if kind in ("box down component", "capsule end"):
            ok = v >= 1e-3
        elif kind in ("deepest lead", "nearest lead"):
            ok = v >= t
        elif kind == "area lead":
            ok = v >= 0.1
        else:
            ok = abs(v - t) >= 0.1 * thr
        if not ok:
            bad.append((kind, float(v), float(t)))
    return bad


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_numpy_restatement_agrees_with_the_oracle_with_margins(asset_root, ch):
    lib = _lib(asset_root, ch)
    orc = Oracle(CS.CHARS[ch]["args"], asset_root)
    lay = SnapLayout(orc.num_joints)
    shapes = CS.link_shapes(orc)
    wrong = []
    worst = np.inf
    for st in lib:
        orc.set_snapshot(st.snap)
        B, P = orc.collider_frames()
        taps, after = CS.contacts(orc, st.snap)
        for j in range(orc.num_joints):   # every link: the test link's branch, and no point on any other
            shape, he, thr = shapes[j]
            tap, m64, dec = CS.collide64(B[j], P[j], shape, he, thr, _mani(lay, st.snap, j))
            if tap != tuple(int(x) for x in taps[0, j]):
                wrong.append("%s link %d: numpy %s, oracle %s" % (st, j, tap, tuple(taps[0, j])))
            if j != st.link:
                if min(v for k, v, t in dec if k == "vertex distance") < 2.0 * thr:
                    wrong.append("%s link %d: support vertex within 2 thresholds of the plane" % (st, j))
                continue
            bad = _margins(dec, thr)
            if bad:
                wrong.append("%s: decisions without margin %s" % (st, bad))
            worst = min(worst, min(abs(v - t) / thr for k, v, t in dec if k in ("vertex distance", "cache match", "refresh distance", "lateral drift")))
            # the new point and the refresh: the manifold after the first sub-step as numpy computes it, within fp32 of the oracle's
            # state after both sub-steps for what the second sub-step does not rewrite (lifetimes, impulses of kept points)
            mo = _mani(lay, after, j)
            n = tap[CS.COUNT]
            if st.expect2 is not None and st.expect2[0] == CS.NONE and taps[1, j, CS.COUNT] == n:
                if not np.array_equal(mo[:n, 11], m64[:n, 11] + 1):
                    wrong.append("%s: lifetimes %s, numpy %s + 1" % (st, mo[:n, 11], m64[:n, 11]))
                if np.abs(mo[:n, 1:7] - m64[:n, 1:7]).max(initial=0.0) > 1e-5:
                    wrong.append("%s: cached points moved: %s" % (st, np.abs(mo[:n, 1:7] - m64[:n, 1:7]).max()))
    print("%s: %d states, smallest distance margin %.3f thresholds" % (ch, len(lib), worst))
    assert not wrong, "\n".join(wrong[:20])


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_second_substep_taps_are_robust_to_rounding_noise(asset_root, ch):
    lib = _lib(asset_root, ch)
    orc = Oracle(CS.CHARS[ch]["args"], asset_root)
    lay = SnapLayout(orc.num_joints)
    rng = np.random.default_rng(5)
    moved = []
    for st in lib:
        ref, _ = CS.contacts(orc, st.snap)
        for _ in range(16):
            taps, _ = CS.contacts(orc, perturb(lay, st.snap, rng, rel=4 * 2.0 ** -24))
            if not np.array_equal(taps, ref):
                moved.append(str(st))
                break
    assert not moved, moved


def test_release_state_leaves_and_reenters_the_threshold_within_a_launch(asset_root):
    for ch in CS.CHARS:
        orc = Oracle(CS.CHARS[ch]["args"], asset_root)
        for st in (s for s in _lib(asset_root, ch) if s.cls == "release"):
            orc.set_snapshot(st.snap)
            ev = []
            for _ in range(CS.RELEASE_UPDATES):
                orc.update(CS.DT)
                ev += [tuple(t[st.link, [CS.EVENT, CS.COUNT]]) for t in orc.last_contacts()]
            first = next(i for i, e in enumerate(ev) if e[0] != CS.NONE)
            print("%s %s: points removed in sub-step 1, a new point in sub-step %d of %d" % (ch, st, first + 1, len(ev)))
            assert ev[0] == (CS.NONE, 0)
            assert 10 <= first <= len(ev) - 20 and ev[first][0] == CS.ADD


@pytest.mark.parametrize("ch", list(CS.CHARS))
def test_contact_library_is_deterministic(asset_root, ch):
    a = CS.build(Oracle(CS.CHARS[ch]["args"], asset_root), asset_root, ch)
    b = _lib(asset_root, ch)
    assert [s.name for s in a] == [s.name for s in b]
    assert all(np.array_equal(x.snap, y.snap) and x.expect == y.expect for x, y in zip(a, b))
