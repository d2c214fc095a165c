"""Pins the oracle back-end (oracle/orc_ba.*) on the reference's own code (oracle/_ref) on windows whose float accumulators cross the 1000-update tier
(tests/ba_tiers.py): the order of shiftUp inside AccumulatorApprox::update (before the TopRight / BotRight adds), the `> 1000` test, one counter per
accD(h,t1,t2) / accE / accEB / accHcc / accbc, which residuals and points are counted.  test_ref_pin_ba.py's windows stay below the tier; a float64 bound
(tests/ba_acc_fp64.py) cannot see the order of a tier shift either, only a bit-for-bit comparison can.

On every tier window: the counts the window was built for, the residuals' activity, accumulate() (HA, bA, Hsc, bsc) and solveSystem(0, lambda) (HS, bS) bit for
bit, the step x at 1e-9 (it passes through the reference's Eigen stand-ins, see test_ref_pin_ba.py).  On the schur window, the marginalisation window, also
flagPointsForRemoval -> marginalizePointsF (mode 2 of the accumulators, crossing in pair (1 -> 0) and in accD(1,0,2)): status, res_toZeroF and the prior HM / bM bit
for bit.  The two-keyframe windows have no point that could be marginalised (isInlierNew needs three residuals).
The reference's results are stored in tests/golden/ref_pin_ba_tiers.npz; SDV_RECORD_REF_GOLDEN=1 re-records them.  The device replays the same steps against the
same golden (tests/test_gpu_ba_tiers.py) through golden_same()."""
import numpy as np
import pytest
import ref
import ba_tiers as T
from ref_golden import RefPin

LAM = 0.1
PIN_TEST = "test_tier_window_bit_exact"
PIN_ORDER = ("levels", "active", "HA", "bA", "Hsc", "bsc", "HS", "bS", "x", "HdiF", "bdSumF", "status", "res_to_zero", "HM", "bM")   # golden entries, in order


def golden(name):
    """the stored reference results of one tier window: a RefPin that only reads"""
    return RefPin("pin_ba_tiers", f"{PIN_TEST}[{name}]")


def golden_same(pin, step, mine):
    """`mine` equals the reference's `step` of the window bit for bit"""
    pin.i = PIN_ORDER.index(step)
    return pin.same(mine, None)


def golden_value(pin, step):
    pin.i = PIN_ORDER.index(step)
    return pin.value(None)


def linearized_res_to_zero(r2z, is_linearized):
    """res_toZeroF of the residuals fixLinearizationF ran on, 0 elsewhere (the others hold stale values)"""
    return np.where(np.asarray(is_linearized)[:, None] != 0, r2z, np.float32(0))


@pytest.fixture
def pin(request):
    p = RefPin("pin_ba_tiers", request.node.name); yield p; p.save()


def _at(pin, step):
    assert pin.i == PIN_ORDER.index(step), (pin.i, step)


@pytest.mark.parametrize("name", T.NAMES)
def test_tier_window_bit_exact(name, pin):
    from sdv_loam_b200 import synth
    win, frames = T.window(name); seq = T.sequence(); K, wh = synth.KITTI_K, synth.KITTI_WH
    _at(pin, "levels"); L = int(pin.value(lambda: ref.set_calib(wh[0], wh[1], K)))
    assert L == T.LEVELS
    rf = pin.live(lambda: [ref.Frame(seq.images[k], wh, L) for k in win["kf_idx"]])
    ob = T.linearized(win, frames); rb = pin.live(lambda: ref.BAWindow(win, rf))
    pin.live(lambda: (rb.reset_oob(), rb.linearizeAll(False), rb.applyRes()))
    rs = ob.residuals(); T.check_counts(name, win, rs["active"], rs["new_state"])
    _at(pin, "active"); assert pin.same(rs["active"], lambda: rb.residuals()["active"])
    A = ob.accumulate(); B = pin.live(lambda: rb.accumulate())
    for i, nm in enumerate(("HA", "bA", "Hsc", "bsc")):
        _at(pin, nm); assert pin.same(A[i], lambda: B[i]), nm
    x, HS, bS = ob.solveSystem(0, LAM); r = pin.live(lambda: rb.solveSystem(0, LAM))
    _at(pin, "HS"); assert pin.same(HS, lambda: r[1]), "HS"
    _at(pin, "bS"); assert pin.same(bS, lambda: r[2]), "bS"
    _at(pin, "x"); xr = pin.value(lambda: r[0])
    assert np.allclose(x, xr, rtol=1e-9, atol=1e-9 * np.abs(xr).max()), np.abs(x - xr).max()
    pa = ob.points(); pr = pin.live(lambda: rb.points())
    for k in ("HdiF", "bdSumF"):
        _at(pin, k); assert pin.same(pa[k], lambda: pr[k]), k
    if name != "schur":
        return
    sel = T.marg_selection(win)
    st = ob.flagPointsForRemoval(sel)
    _at(pin, "status"); assert pin.same(st, lambda: rb.flagPointsForRemoval(sel))
    T.check_marg_counts(win, ob.residuals()["active"], st)
    _at(pin, "res_to_zero"); assert pin.same(linearized_res_to_zero(*ob.res_to_zero()), lambda: linearized_res_to_zero(*rb.res_to_zero()))
    ob.marginalizePointsF(st); pin.live(lambda: rb.marginalizePointsF())
    HM, bM = ob.prior(); P = pin.live(lambda: rb.prior())
    _at(pin, "HM"); assert pin.same(HM, lambda: P[0]), "HM"
    _at(pin, "bM"); assert pin.same(bM, lambda: P[1]), "bM"
