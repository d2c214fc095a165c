"""The oracle back-end (orc.BAWindow) against the float64 restatements of tests/ba_fp64.py on the three LIVE windows of tests/golden/seq_ba_ref.npz (the reference's own
running pipeline: seven keyframes without frameID 0, a prior of real marginalisations with cond ~1e9, intrinsics ~1e-6 away from value_zero) and on one synthetic
window (frameID 0, a moved value_zero): calcMEnergy, the assembled system and the step of solveSystem at iterations 0 and 2, and the keyframe hand-over.  On every
live window the same restatement with value_zero := value falls outside the bounds, so these checks see a back-end that lost CalibHessian::value_zero.  CPU only."""
import os
import numpy as np
import pytest
import orc
import ba_fp64 as F
from conftest import SMALL_K, SMALL_WH, cached_sequence

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seq_ba_ref.npz")
WINDOW_KEYS = ("nF", "kf_idx", "T_eval", "state", "state_zero", "ab_exposure", "frameID", "frameEnergyTH", "K", "K_zero", "uv", "idepth", "idepth_zero", "color", "weights", "host",
               "hasDepthPrior", "isFromSensor", "res_begin", "r_point", "r_host", "r_target", "r_hasMatcher", "r_matcher", "r_isNew", "HM", "bM")
LAM = 0.1                                                                    # the first lambda of FullSystem::optimize (FullSystemOptimize.cpp:391)


def live_windows(wh):
    """{frame of the reference run: window dict} of tests/golden/seq_ba_ref.npz, and its pyramid levels"""
    g = np.load(GOLD); out = {}
    for i in g["windows"]:
        p = f"w{i}_"; A = {k: g[p + k] for k in WINDOW_KEYS}; A["nF"] = int(A["nF"]); A["kf_idx"] = [int(k) for k in A["kf_idx"]]; A["wh"] = wh
        out[int(i)] = A
    return out, int(g["levels"])


def select(win, marg_host, every):
    """the points flagged at a keyframe step: those of the frame about to be eliminated plus every k-th, never the newest keyframe's (FullSystem.cpp:751)"""
    sel = (np.asarray(win["host"]) == marg_host).astype(np.int32); sel[::every] = 1
    sel[np.asarray(win["host"]) == win["nF"] - 1] = 0
    return sel


@pytest.fixture(scope="module")
def cases():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import synth
    seq = cached_sequence(200, 1000, synth.KITTI_K, synth.KITTI_WH, step=0.5)
    wins, L = live_windows(seq.wh); out = {}
    for i, w in wins.items():
        out[f"live{i}"] = (w, [orc.Frame(seq.images[k], L) for k in w["kf_idx"]])
    s5 = cached_sequence(5, 3000, SMALL_K, SMALL_WH)
    w = synth.make_ba_window(s5, [0, 1, 2, 3, 4], n_per_frame=120, seed=5, pose_noise=(0.004, 0.0003), match_noise=0.15, prior_scale=1e-2)
    w["K_zero"] = F.calib_value(w) * (1 + 1e-4 * np.random.default_rng(8).normal(size=4))
    out["synthetic"] = (w, [orc.Frame(s5.images[k], 4) for k in w["kf_idx"]])
    return out


CASES = ["live27", "live36", "live45", "synthetic"]


@pytest.mark.parametrize("case", CASES)
def test_calc_m_energy(cases, case):
    win, frames = cases[case]
    ob = orc.BAWindow(win, frames); HM, bM = np.asarray(win["HM"], np.float64), np.asarray(win["bM"], np.float64)
    d = F.stitched_delta(win, ob.frames()); e, bnd = F.calc_m_energy(HM, bM, d)
    eo = ob.calcMEnergy()
    assert abs(eo - e) <= 2 * bnd, (case, eo, e, bnd)
    lost, _ = F.calc_m_energy(HM, bM, F.stitched_delta(F.without_value_zero(win), ob.frames()))
    assert abs(eo - lost) > 2 * bnd, (case, eo, lost, bnd)                    # teeth: a lost value_zero is visible


@pytest.mark.parametrize("case", CASES)
def test_solve_system_iterations_0_and_2(cases, case):
    win, frames = cases[case]
    ob = orc.BAWindow(win, frames); HM, bM = np.asarray(win["HM"], np.float64), np.asarray(win["bM"], np.float64)
    ob.reset_oob(); ob.linearizeAll(False); ob.applyRes()
    system = ob.accumulate()
    x0, HS, bS = ob.solveSystem(0, LAM)
    d = F.stitched_delta(win, ob.frames())
    bS_ref, bnd = F.check_assembly(HS, bS, system, HM, bM, d, case)
    F.check_backward_error(x0, HS, bS, LAM, what=case)
    _, bS_lost, _ = F.assemble(*system, HM, bM, F.stitched_delta(F.without_value_zero(win), ob.frames()))
    assert np.any(np.abs(bS - bS_lost) > 2 * bnd), case                       # teeth: a lost value_zero is visible in bS
    x2, HS2, bS2 = ob.solveSystem(2, LAM)
    assert np.array_equal(HS2, HS) and np.array_equal(bS2, bS), case
    F.check_orthogonalized(x0, x2, ob.frames()["T_eval"], case)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("where", ["first", "middle"])
def test_keyframe_hand_over(cases, case, where):
    win, frames = cases[case]
    ob = orc.BAWindow(win, frames); ob.optimize(6)
    idx = 0 if where == "first" else win["nF"] // 2
    st = ob.flagPointsForRemoval(select(win, idx, 3)); assert (st == 2).sum() > 30, case
    HM0, bM0 = ob.prior(); m = ob.marginalizePointsF(st); HM1, bM1 = ob.prior()
    rs = ob.residuals(); r2z, _ = ob.res_to_zero()
    dense = F.dense_marg_system(win, rs["efJ"], r2z, rs["active"], ob.precalc, st)
    F.check_marginalized_points(win, m, HM0, bM0, HM1, bM1, dense, case)
    state = ob.frames()["state"][idx]
    ob.marginalizeFrame(idx); H2, b2 = ob.prior()
    F.check_marginalized_frame(H2, b2, HM1, bM1, idx, int(win["frameID"][idx]), state, case)
