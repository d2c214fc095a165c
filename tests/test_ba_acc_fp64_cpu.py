"""The oracle back-end's float accumulators against the float64 restatement of tests/ba_acc_fp64.py, entry by entry within their tier-aware bounds: HA / bA / Hsc / bsc
of accumulate() and M / Mb / Msc / Mbsc of marginalizePointsF, on the three LIVE windows of tests/golden/seq_ba_ref.npz and the synthetic window of
test_ba_fp64_cpu.py, and on the tier windows of tests/ba_tiers.py, whose accumulators cross the 1000-update tier.  The update counts the restatement finds equal
those of ba_tiers.count_updates.  Three mistaken restatements fall outside the bounds: one that counts an inactive residual (the live windows hold none: the
reference had dropped them), one that lets LiDAR points into the Schur complement, one whose finish() loses the completed 1000-update chunks (only where a bucket
crossed the tier; below it the variant is the correct result).  The bounds cannot see the order of a tier shift: test_ref_pin_ba_tiers.py pins that.  CPU only."""
import numpy as np
import pytest
import ba_acc_fp64 as A
import ba_tiers
from test_ba_fp64_cpu import CASES, LAM, cases, select  # noqa: F401  (cases: the module fixture of the live and synthetic windows)
from tracker_fp64 import Report

VARIANTS = ("inactive", "lidar", "lost_tiers")


def _teeth(win, eq, got, args, kw, what):
    """each mistaken restatement of normal_equations() is rejected somewhere: in a top accumulator's quantity for "inactive" (the Hessian at least: marginalizePointsF's
    res_toZeroF of a residual that was never linearised is stale), in a Schur one for "lidar", and for "lost_tiers" some quantity exactly when a bucket crossed
    the tier"""
    top, sc = list(eq[0])[:2], list(eq[0])[2:]
    crossed = any(n > 1000 for c in ("top", "D", "E") for n in eq[1][c].values()) or eq[1]["hcc"] > 1000
    inactive = (np.asarray(args[0]["active"]) == 0) & ((np.asarray(kw["status"])[np.asarray(win["r_point"])] == 2) if "status" in kw else True)
    for v in VARIANTS:
        if v == "inactive" and not inactive.any():
            assert what.startswith("live") and "status" not in kw, what       # the live windows hold no inactive residual: the reference had dropped them
            continue
        bad = A.rejected(eq, A.normal_equations(win, *args, variant=v, **kw), got)
        if v == "inactive":
            assert set(top) & set(bad), (what, v, bad)
        elif v == "lidar":
            assert set(sc) & set(bad), (what, v, bad)
        else:
            assert bool(bad) == crossed, (what, v, bad, crossed)


def _counts_equal(eq, c):
    return (eq[1]["top"], eq[1]["D"], eq[1]["E"], eq[1]["hcc"]) == (c["top"], c["D"], c["E"], c["hcc"])


def _accumulate_case(win, frames, what, rep):
    ob = ba_tiers.linearized(win, frames); rs = ob.residuals()
    got = dict(zip(("HA", "bA", "Hsc", "bsc"), ob.accumulate()))
    args = (rs, ob.points(), ob.precalc, ob.frames()); eq = A.normal_equations(win, *args)
    A.check_equations(eq, got, what, rep)
    assert _counts_equal(eq, ba_tiers.count_updates(win, rs["active"])), what
    _teeth(win, eq, got, args, {}, what)
    return eq, rs


def _hand_over(ob, win, sel, what, rep):
    """flagPointsForRemoval -> marginalizePointsF: M / Mb / Msc / Mbsc within the bounds, the prior update bit-exact, the mistaken restatements rejected"""
    st = ob.flagPointsForRemoval(sel)
    HM0, bM0 = ob.prior(); m = ob.marginalizePointsF(st); HM1, bM1 = ob.prior()
    rs = ob.residuals(); r2z, _ = ob.res_to_zero()
    dense = A.dense_marg_system(win, rs["efJ"], r2z, rs["active"], ob.precalc, st)
    A.check_marginalized_points(win, m, HM0, bM0, HM1, bM1, dense, what, rep)
    assert _counts_equal(dense, ba_tiers.count_updates(win, rs["active"], st)), what
    _teeth(win, dense, m, (rs, None, ob.precalc), dict(status=st, res_to_zero=r2z), what)
    return st, rs


@pytest.mark.parametrize("case", CASES)
def test_accumulators_within_bounds(cases, case):
    win, frames = cases[case]; rep = Report(f"accumulate {case}")
    eq, _ = _accumulate_case(win, frames, case, rep)
    assert max(eq[1]["top"].values()) <= 1000, case                                # these windows stay below the tier
    rep.print()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("where", ["first", "middle"])
def test_marginalized_points_within_bounds(cases, case, where):
    """the keyframe hand-over of test_ba_fp64_cpu.py::test_keyframe_hand_over, M / Mb / Msc / Mbsc held to the derived bounds"""
    import orc
    win, frames = cases[case]; rep = Report(f"marginalizePointsF {case} {where}")
    ob = orc.BAWindow(win, frames); ob.optimize(6)
    idx = 0 if where == "first" else win["nF"] // 2
    st, _ = _hand_over(ob, win, select(win, idx, 3), case, rep)
    assert (st == 2).sum() > 30, case
    rep.print()


@pytest.fixture(scope="module")
def tier_cases():
    return {n: ba_tiers.window(n) for n in ba_tiers.NAMES}


@pytest.mark.parametrize("name", ba_tiers.NAMES)
def test_accumulators_within_bounds_tier_windows(tier_cases, name):
    win, frames = tier_cases[name]; rep = Report(f"accumulate {name}")
    _, rs = _accumulate_case(win, frames, name, rep)
    ba_tiers.check_counts(name, win, rs["active"], rs["new_state"])
    rep.print()


def test_marginalized_points_tier_window(tier_cases):
    """marginalizePointsF (mode 2 of the accumulators) on the schur window: pair (1 -> 0) and accD(1,0,2) cross 1000"""
    win, frames = tier_cases["schur"]; rep = Report("marginalizePointsF schur")
    ob = ba_tiers.linearized(win, frames); ob.solveSystem(0, LAM)
    st, rs = _hand_over(ob, win, ba_tiers.marg_selection(win), "schur", rep)
    ba_tiers.check_marg_counts(win, rs["active"], st)
    rep.print()
