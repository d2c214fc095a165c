"""GPU (-m gpu) counterpart of tests/test_sequence_ba.py: the device back-end on the three LIVE windows of the reference's own run (tests/golden/seq_ba_ref.npz:
seven keyframes without frameID 0, ~1 100 points of which ~750 from LiDAR, a prior of real marginalisations with cond ~1e9, intrinsics that left value_zero).  The 15
distinct keyframe images are ingested once and the windows share those frame handles.  Single-window entries (sdv_ba_set_window + sdv_ba_set_calib_zero +
sdv_ba_set_points) and batched ones (sdv_ba_set_window_batch with calib_value_zero, windows at non-contiguous indices): energies, the assembled system and the step
at iterations 0 and 2, optimize(6) and the keyframe hand-over bit-exact against the oracle, within the float64 bounds of tests/ba_fp64.py, and optimize(6) within
the reference's stored results at the bounds test_sequence_ba.py uses."""
import numpy as np
import pytest
import orc
import ba_fp64 as F
from conftest import cached_sequence
from test_ba_fp64_cpu import GOLD, LAM, live_windows, select

pytestmark = pytest.mark.gpu


def _bit(a, b, what):
    """a and b identical (NaN equal to NaN); on a mismatch, the first differing entry"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a, b, equal_nan=True):
        eq = (a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else a == b
        k = np.unravel_index(int(np.argmin(eq)), a.shape)
        raise AssertionError(f"{what}: first difference at {k}: device {a[k]!r}, oracle {b[k]!r}")


@pytest.fixture(scope="module")
def world():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    seq = cached_sequence(200, 1000, synth.KITTI_K, synth.KITTI_WH, step=0.5)
    wins, L = live_windows(seq.wh)
    imgs = sorted({k for w in wins.values() for k in w["kf_idx"]})
    assert len(imgs) == 15
    ctx = api.Context(synth.KITTI_K, *seq.wh, levels=L, max_frames=24, max_kf_images=24)
    for k in imgs:                                                           # frame handle = image index; windows share handles
        ctx.makeImages(k, seq.images[k])
    frames = {k: orc.Frame(seq.images[k], L) for k in imgs}
    yield api, ctx, wins, frames, np.load(GOLD)
    ctx.close()


def _oracle(win, frames):
    return orc.BAWindow(win, [frames[k] for k in win["kf_idx"]])


def _optimized_like_oracle(e, ob, r, ro, what):
    assert (r["iterations"], r["accepts"]) == (ro["iterations"], ro["accepts"]), (what, r, ro)
    _bit(np.float32(r["rmse"]), np.float32(ro["rmse"]), f"{what} rmse")
    fg, fo = e.frames(), ob.frames()
    for k in ("T_eval", "state", "frameEnergyTH"):
        _bit(fg[k], fo[k], f"{what} {k}")
    _bit(fg["calib_value"], ob.calib()[0], f"{what} calib_value")
    _bit(e.points()["idepth"], ob.points()["idepth"], f"{what} idepth")
    sg, so = e.residuals(), ob.residuals()
    _bit(sg["state"], so["state"], f"{what} residual state"); _bit(sg["toRemove"], so["toRemove"], f"{what} toRemove")


def _within_reference(g, i, e, r):
    """the bounds of test_sequence_ba.py against the reference's own optimize(6) of the window"""
    p = f"w{i}_"; rmse_ref = float(g[p + "rmse"])
    assert abs(float(r["rmse"]) - rmse_ref) <= 1e-6 * rmse_ref, (i, r["rmse"], rmse_ref)
    fg = e.frames()
    assert np.abs(e.points()["idepth"] - g[p + "after_idepth"]).max() < 1e-6 and np.abs(fg["state"] - g[p + "after_state"]).max() < 1e-6, i
    assert np.abs(fg["calib_value"] * np.array([50, 50, 50, 50]) - g[p + "after_K"]).max() < 1e-5 * 700, i


def test_single_window_energies_and_solve(world):
    api, ctx, wins, frames, g = world
    for j, (i, win) in enumerate(wins.items()):
        e = api.EnergyFunctional(ctx, win, win["kf_idx"], window=j); ob = _oracle(win, frames)
        HM, bM = np.asarray(win["HM"], np.float64), np.asarray(win["bM"], np.float64)
        EL, EM = e.energies()
        _bit(EL, ob.calcLEnergy(), f"w{i} calcLEnergy"); _bit(EM, ob.calcMEnergy(), f"w{i} calcMEnergy")
        d = F.stitched_delta(win, e.frames()); em, bnd = F.calc_m_energy(HM, bM, d)
        assert abs(EM - em) <= 2 * bnd, (i, EM, em, bnd)
        e.reset_oob(); e.linearizeAll(False); e.applyRes(); ob.reset_oob(); ob.linearizeAll(False); ob.applyRes()
        system_o = ob.accumulate()
        x0, HS, bS, system = e.solveSystem(0, LAM); xo, HSo, bSo = ob.solveSystem(0, LAM)
        for name, a, b in zip(("HA", "bA", "Hsc", "bsc"), system, system_o):
            _bit(a, b, f"w{i} it0 {name}")
        _bit(HS, HSo, f"w{i} it0 HS"); _bit(bS, bSo, f"w{i} it0 bS"); _bit(x0, xo, f"w{i} it0 x")
        F.check_assembly(HS, bS, system, HM, bM, d, f"w{i}")
        F.check_backward_error(x0, HS, bS, LAM, what=f"w{i}")
        x2, HS2, bS2, _ = e.solveSystem(2, LAM); xo2, _, _ = ob.solveSystem(2, LAM)
        _bit(HS2, HS, f"w{i} it2 HS"); _bit(bS2, bS, f"w{i} it2 bS"); _bit(x2, xo2, f"w{i} it2 x")
        F.check_orthogonalized(x0, x2, e.frames()["T_eval"], f"w{i}")


def test_single_window_optimize_and_hand_over(world):
    api, ctx, wins, frames, g = world
    for j, (i, win) in enumerate(wins.items()):
        e = api.EnergyFunctional(ctx, win, win["kf_idx"], window=3 + j); ob = _oracle(win, frames)
        r, ro = e.optimize(6), ob.optimize(6)
        _optimized_like_oracle(e, ob, r, ro, f"w{i}"); _within_reference(g, i, e, r)
        _hand_over([e], [ob], [win], [(0, 3), (win["nF"] // 2, 4), (1, 5)][j], f"w{i} single")


def test_batched_install_optimize_and_hand_over(world):
    api, ctx, wins, frames, g = world
    W = [9, 6, 13]                                                           # non-contiguous, not in order
    ws = list(wins.values())
    eb = api.EnergyFunctional.install_batch(ctx, W, ws, [w["kf_idx"] for w in ws])
    obs = [_oracle(w, frames) for w in ws]
    for e, ob, (i, w) in zip(eb, obs, wins.items()):                         # K_zero carried by sdv_ba_set_window_batch
        EL, EM = e.energies()
        _bit(EL, ob.calcLEnergy(), f"w{i} batch calcLEnergy"); _bit(EM, ob.calcMEnergy(), f"w{i} batch calcMEnergy")
    r = api.optimize_batch(ctx, W, 6)
    for k, (e, ob, (i, w)) in enumerate(zip(eb, obs, wins.items())):
        rk = dict(rmse=r["rmse"][k], iterations=int(r["iterations"][k]), accepts=int(r["accepts"][k]))
        _optimized_like_oracle(e, ob, rk, ob.optimize(6), f"w{i} batch"); _within_reference(g, i, e, rk)
    _hand_over(eb, obs, ws, [(w["nF"] // 2, 3 + k) for k, w in enumerate(ws)], "batch", api=api)


def _hand_over(es, obs, ws, plan, what, api=None):
    """flagPointsForRemoval -> marginalizePointsF -> marginalizeFrame(idx) on optimised windows: status, res_toZeroF, M / Mb / Msc / Mbsc and the priors
    bit-exact against the oracle and within the ba_fp64 bounds.  api: through the batched entries; plan: (idx, every) per window, or one pair"""
    if isinstance(plan, tuple):
        plan = [plan]
    sels = [select(w, idx, every) for w, (idx, every) in zip(ws, plan)]
    sts = api.flag_points_batch(es, sels) if api else [e.flagPointsForRemoval(s) for e, s in zip(es, sels)]
    priors0 = [e.prior() for e in es]
    if api:
        api.marginalize_points_batch(es); ms = []
        for e in es:
            n = e.n; M = np.zeros((n, n)); Mb = np.zeros(n); S = np.zeros((n, n)); Sb = np.zeros(n)
            e._sel(); e.ctx._ck(api.LIB.sdv_ba_get_system(e.ctx.p, M, Mb, S, Sb, np.zeros((n, n)), np.zeros(n)))
            ms.append(dict(M=M, Mb=Mb, Msc=S, Mbsc=Sb))
    else:
        ms = [e.marginalizePointsF() for e in es]
    states = [e.frames()["state"][idx] for e, (idx, _) in zip(es, plan)]
    for e, ob, w, st, sel, m, (HM0, bM0), (idx, _) in zip(es, obs, ws, sts, sels, ms, priors0, plan):
        tag = f"{what} window {e.window}"
        so = ob.flagPointsForRemoval(sel); _bit(st, so, f"{tag} status")
        assert (st == 2).sum() > 30, tag
        HMo0, bMo0 = ob.prior(); _bit(HM0, HMo0, f"{tag} HM before"); _bit(bM0, bMo0, f"{tag} bM before")
        mo = ob.marginalizePointsF(so)
        r2z, lin = e.linearized(); r2zo, lino = ob.res_to_zero()
        _bit(lin, lino, f"{tag} isLinearized"); _bit(r2z, r2zo, f"{tag} res_toZeroF")
        for k in ("M", "Mb", "Msc", "Mbsc"):
            _bit(m[k], mo[k], f"{tag} {k}")
        HM1, bM1 = e.prior(); HMo1, bMo1 = ob.prior(); _bit(HM1, HMo1, f"{tag} HM after points"); _bit(bM1, bMo1, f"{tag} bM after points")
        rs = e.residuals()
        F.check_marginalized_points(w, m, HM0, bM0, HM1, bM1, F.dense_marg_system(w, rs["efJ"], r2z, rs["active"], e.precalc, st), tag)
    if api:
        pa = api.marginalize_frames_batch(es, [[idx] for idx, _ in plan])
    else:
        for e, (idx, _) in zip(es, plan):
            e.marginalizeFrame(idx)
        pa = [e.prior() for e in es]
    for e, ob, w, (H2, b2), (HM1, bM1), (idx, _), state in zip(es, obs, ws, pa, [ob.prior() for ob in obs], plan, states):
        tag = f"{what} window {e.window} frame {idx}"
        ob.marginalizeFrame(idx); Ho, bo = ob.prior()
        _bit(H2, Ho, f"{tag} HM"); _bit(b2, bo, f"{tag} bM")
        F.check_marginalized_frame(H2, b2, HM1, bM1, idx, int(w["frameID"][idx]), state, tag)
