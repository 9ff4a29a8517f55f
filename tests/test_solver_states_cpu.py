"""The constructed state library (tests/solver_states.py) reaches, in the CPU oracle, every branch of the constraint solve it was built for:
each storage bucket of solve_rows (none, <= W, <= kSq2, packed, overflow), shallow and deep joint-limit rows, the limit impulse at its cap,
the coordinate clamp in the unconstrained update and after PGS, friction rows skipped for a point whose normal impulse is 0, and
HasVelExploded.  Without this check the library could decay into states that exercise nothing.  Branches no physically meaningful state
of a character reaches are listed by name in UNREACHABLE, with the reason."""
import numpy as np
import pytest

from tests import solver_states as S
from tests.oracle_binding import Oracle

# The dog's limited joints (forearms, legs) are light: even at the 100 rad/s coordinate clamp the impulse that stops one of them stays
# below 45 (1 / (M^-1)_jj < 0.45), so its limit rows never reach maxAppliedImpulse = 100.
UNREACHABLE = {("dog3d", "limit impulse at the cap")}


def reached(orc, asset_root, ch):
    """{branch name: [state names that reach it]} over the library of character ch, and the per-state rows"""
    o2 = Oracle(S.CHARS[ch]["args"], asset_root)
    lib = S.build(orc, asset_root, ch)
    hit = {}
    for st in lib:
        r, _ = S.last_rows(o2, st.snap)
        rows = int(r[-1, S.LIMITS] + 3 * r[-1, S.POINTS])
        names = ["%s: %s rows" % (st.cls, S.BUCKETS[S.bucket(rows, ch)])]
        if r[:, S.LIMITS].sum() > r[:, S.LIMIT_DEEP].sum():
            names.append("shallow limit row")
        if r[:, S.LIMIT_DEEP].any():
            names.append("deep limit row (split impulse)")
        if r[:, S.LIMIT_SAT].any():
            names.append("limit impulse at the cap")
        if r[:, S.CLAMP_ABA].any():
            names.append("clamp in the unconstrained update")
        if r[:, S.CLAMP_PGS].any():
            names.append("clamp after PGS")
        if r[:, S.FRICTION_SKIP].any():
            names.append("friction rows skipped")
        if not o2.check_valid_episode():
            names.append("HasVelExploded")
        for n in names:
            hit.setdefault(n, []).append(st.name)
    return lib, hit


def expected(ch):
    """branch name -> the class whose states must reach it"""
    e = {"stance: %s rows" % b: "stance" for b in S.BUCKETS}
    e.update({"free: none rows": "free", "shallow limit row": "limit", "deep limit row (split impulse)": "limit", "limit impulse at the cap": "limit",
              "clamp in the unconstrained update": "clamp", "clamp after PGS": "clamp", "friction rows skipped": "release", "HasVelExploded": "explode"})
    return e


@pytest.mark.parametrize("ch", list(S.CHARS))
def test_every_state_class_reaches_its_branch_in_the_oracle(asset_root, ch):
    orc = Oracle(S.CHARS[ch]["args"], asset_root)
    lib, hit = reached(orc, asset_root, ch)
    by_name = {st.name: st.cls for st in lib}
    missing = []
    print("%s: %d constructed states" % (ch, len(lib)))
    for branch, cls in expected(ch).items():
        states = [n for n in hit.get(branch, []) if branch.startswith("stance") or by_name[n] == cls]
        if (ch, branch) in UNREACHABLE:
            print("  %-36s unreachable for %s (see UNREACHABLE); reached by %d states" % (branch, ch, len(states)))
            assert not states, "%s is listed as unreachable for %s but %s reach it" % (branch, ch, states[:3])
            continue
        print("  %-36s %3d states of class %-8s e.g. %s" % (branch, len(states), cls, states[0] if states else "-"))
        if not states:
            missing.append(branch)
    assert not missing, "%s: no %s state reaches %s" % (ch, "/".join(sorted(set(expected(ch)[b] for b in missing))), missing)


@pytest.mark.parametrize("ch", list(S.CHARS))
def test_state_library_is_deterministic(asset_root, ch):
    a = S.build(Oracle(S.CHARS[ch]["args"], asset_root), asset_root, ch)
    b = S.build(Oracle(S.CHARS[ch]["args"], asset_root), asset_root, ch)
    assert [s.name for s in a] == [s.name for s in b]
    assert all(np.array_equal(x.snap, y.snap) for x, y in zip(a, b))
