"""float64 restatements of the back-end's prior terms (OptimizationBackend/EnergyFunctional.cpp), for checking the oracle (orc.BAWindow) on the CPU and the device
(api.EnergyFunctional) on the GPU with the same code.  Every function takes plain arrays: the window dict (synth.make_ba_window's layout, or a live window of
tests/golden/seq_ba_ref.npz) and what frames() / solveSystem() / residuals() / precalc() / prior() of either back-end return.

Bounds: a float64 sum or product of n terms, however ordered, is within gamma(n) * sum |terms| of the exact value (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., section 3.1); two evaluations in different orders are within twice that of each other.  Each check states its bound beside it, taken from the
actual terms.  The float-accumulated marginalisation blocks M / Msc are compared with the tolerances tests/test_oracle_marg.py uses."""
import numpy as np

U = 2.0 ** -53
SF = np.float64(np.float32(1) / np.float32(50))        # CalibHessian::value = value_scaled * (1.0f/50.0f), a float factor times a double (CalibHessian::setValueScaled)
SCALE_XI_TRANS, SCALE_XI_ROT = 0.5, 1.0                # HessianBlocks.h:34-35
MARG_WEIGHT = 0.5 * 0.5                                # setting_margWeightFac (settings.cpp:71)
TRANS_PRIOR, ROT_PRIOR = 1e10, 1e11                    # setting_initialTransPrior / RotPrior (settings.cpp:23-24): FrameHessian::getPrior of frameID 0


def gamma(n):
    return n * U / (1 - n * U)


def calib_value(win):
    """CalibHessian::value of a freshly installed window"""
    return np.asarray(win["K"], np.float64) * SF


def stitched_delta(win, frames, value=None):
    """getStitchedDeltaF (EnergyFunctional.h): [cDeltaF = float(value - value_zero) as double (EnergyFunctional.cpp:144), (state - state_zero)[:6] per frame].
    value: CalibHessian::value (default: that of a fresh install); value_zero: win["K_zero"], or value itself when the window has none."""
    v = calib_value(win) if value is None else np.asarray(value, np.float64)
    vz = np.asarray(win["K_zero"], np.float64) if "K_zero" in win else v
    st = np.asarray(frames["state"], np.float64); st0 = np.asarray(win["state_zero"], np.float64)
    return np.concatenate([(v - vz).astype(np.float32).astype(np.float64), (st - st0)[:, :6].reshape(-1)])


def without_value_zero(win):
    """the window as a back-end that lost CalibHessian::value_zero sees it (value_zero = value)"""
    out = dict(win); out.pop("K_zero", None)
    return out


def calc_m_energy(HM, bM, d):
    """calcMEnergy (EnergyFunctional.cpp:284-293): d . (2 bM + HM d), and its bound: each of the n row sums and the final dot product is an fp64 sum of at most
    n + 2 terms, so |computed - exact| <= gamma(2n + 2) * sum_i |d_i| (2 |bM_i| + sum_j |HM_ij d_j|)"""
    n = len(d); Hd = HM @ d
    e = float(d @ (2 * bM + Hd))
    return e, gamma(2 * n + 2) * float(np.abs(d) @ (2 * np.abs(bM) + np.abs(HM) @ np.abs(d)))


def assemble(HA, bA, Hsc, bsc, HM, bM, d):
    """solveSystemF's assembly for the default SOLVER_ORTHOGONALIZE_X_LATER (settings.cpp:34; EnergyFunctional.cpp:668-700, the else branch at :695, no system
    orthogonalisation): HS = (HA + HM) - Hsc elementwise -- bit-exact, as both sides round each of the two fp64 operations the same way --, bS = (bA + (bM + HM d)) - bsc,
    whose only inexact part besides the three rounded additions is the matrix-vector product: bound gamma(n + 3) * (|bA| + |bM| + |HM| |d| + |bsc|) per entry."""
    n = len(d)
    HS = (HA + HM) - Hsc
    bS = (bA + (bM + HM @ d)) - bsc
    return HS, bS, gamma(n + 3) * (np.abs(bA) + np.abs(bM) + np.abs(HM) @ np.abs(d) + np.abs(bsc))


def check_assembly(HS, bS, system, HM, bM, d, what=""):
    """HS bit-exact and bS within twice the bound of assemble() (two evaluations of the same sum, each within the bound of the exact value)"""
    HA, bA, Hsc, bsc = system
    HS_ref, bS_ref, bnd = assemble(HA, bA, Hsc, bsc, HM, bM, d)
    assert np.array_equal(HS, HS_ref), (what, "HS", np.abs(HS - HS_ref).max())
    err = np.abs(bS - bS_ref); k = int(np.argmax(err / (2 * bnd + 1e-300)))
    assert np.all(err <= 2 * bnd), (what, "bS", k, bS[k], bS_ref[k], err[k], 2 * bnd[k])
    return bS_ref, bnd


def lm_matrix(HS, lam):
    """the matrix the step solves: HS with its diagonal scaled by (1 + lambda) (EnergyFunctional.cpp:703), symmetric as its lower triangle.  HS itself is not
    symmetric (the stitched HA and Hsc differ from their transposes by ~1e-10 relative on live windows), and the LDLT reads the lower triangle only: against the
    matrix as given, the residual of the step is several hundred times the fp64 backward-error bound, against the matrix the solver factors it is below 1e-3 of it."""
    Hl = np.tril(HS) + np.tril(HS, -1).T; Hl[np.diag_indices(len(HS))] *= (1 + lam)
    return Hl


def check_backward_error(x, HS, bS, lam, c=1.0, what=""):
    """the step at iteration 0 solves Hl x = bS with a small backward error: ||Hl x - bS|| <= c n 2^-53 (||Hl|| ||x|| + ||bS||) (2-norms).  The solve is a
    Jacobi-scaled, pivoted LDLT of a symmetric positive definite matrix, backward stable; with cond(HS) up to ~1e9 a forward-error check against np.linalg.solve
    would prove little.  Returns the ratio of the residual to the bound without c."""
    Hl = lm_matrix(HS, lam); n = len(x)
    r = np.linalg.norm(Hl @ x - bS); scale = n * U * (np.linalg.norm(Hl, 2) * np.linalg.norm(x) + np.linalg.norm(bS))
    assert r <= c * scale, (what, r, c * scale)
    return r / scale


def nullspaces(T_eval):
    """getNullspaces (FullSystemOptimize.cpp:548-588) as an exact span: per frame, the pose directions Adj(worldToCam_evalPT) e_i and the scale direction (t, 0),
    rows divided by SCALE_XI_TRANS / SCALE_XI_ROT, on the frame rows of the stitched system (the reference takes central differences of the same linear maps)"""
    import orc
    nF = len(T_eval); N = np.zeros((4 + 6 * nF, 7)); sc = np.array([1 / SCALE_XI_TRANS] * 3 + [1 / SCALE_XI_ROT] * 3)
    for f, T in enumerate(T_eval):
        N[4 + 6 * f:10 + 6 * f, :6] = orc.se3_adj(T) * sc[:, None]
        N[4 + 6 * f:7 + 6 * f, 6] = np.asarray(T, np.float64)[4:7] * sc[:3]
    return N


def check_orthogonalized(x0, x2, T_eval, what=""):
    """at iteration >= 2 SOLVER_ORTHOGONALIZE_X_LATER projects the step: x2 = x0 - N N^+ x0 (EnergyFunctional.cpp:615-648).  The removed part lies in the span of
    the nullspaces (relative least-squares residual <= 1e-8: the directions are normalised central differences) and is orthogonal to the step that is kept."""
    N = nullspaces(T_eval); dx = x0 - x2
    assert np.linalg.norm(dx) > 0, what
    coef = np.linalg.lstsq(N, dx, rcond=None)[0]
    assert np.linalg.norm(dx - N @ coef) <= 1e-8 * np.linalg.norm(dx), (what, np.linalg.norm(dx - N @ coef), np.linalg.norm(dx))
    assert abs(dx @ x2) <= 1e-8 * np.linalg.norm(dx) * np.linalg.norm(x2), (what, dx @ x2)


def dense_marg_system(win, efJ, res_to_zero, active, precalc, status):
    """explicit float64 normal equations over [calib(4), frames(6 nF), inverse depths of the PS_MARGINALIZE points] from efJ / res_toZeroF
    (tests/test_oracle_marg.py::dense_marg_system for any window): precalc(h, t) -> dict with adHost / adTarget"""
    nF = int(win["nF"]); N = 4 + 6 * nF
    mp = np.where(np.asarray(status) == 2)[0]; col = {int(p): N + i for i, p in enumerate(mp)}
    H = np.zeros((N + len(mp), N + len(mp))); b = np.zeros(N + len(mp)); ads = {}
    for r in range(len(active)):
        p = int(win["r_point"][r])
        if status[p] != 2 or not active[r]:
            continue
        h, t = int(win["r_host"][r]), int(win["r_target"][r])
        if (h, t) not in ads:
            pc = precalc(h, t); ads[h, t] = (np.asarray(pc["adHost"], np.float64), np.asarray(pc["adTarget"], np.float64))
        aH, aT = ads[h, t]; J = np.asarray(efJ[r], np.float64); Jr = np.zeros((2, N + len(mp)))
        for a in range(2):
            Jx = J[2 + 6 * a: 8 + 6 * a]
            Jr[a, :4] = J[14 + 4 * a: 18 + 4 * a]
            Jr[a, 4 + 6 * h: 10 + 6 * h] += aH @ Jx
            Jr[a, 4 + 6 * t: 10 + 6 * t] += aT @ Jx
            Jr[a, col[p]] = J[22 + a]
        H += Jr.T @ Jr; b += Jr.T @ np.asarray(res_to_zero[r], np.float64)
    prior = np.where(np.asarray(win["hasDepthPrior"]) == 1, 2500.0 * 600 * 600, 0.0)      # the depth prior of test_oracle_marg.py::dense_marg_system
    for p in mp:
        H[col[int(p)], col[int(p)]] += prior[p]
    return H, b, mp, col


def check_marginalized_points(win, m, HM0, bM0, HM1, bM1, dense, what=""):
    """marginalizePointsF (EnergyFunctional.cpp:514-576): M / Mb the frame-calib block of the dense system, Msc / Mbsc its Schur complement over the vision points
    (LiDAR points never reach the Schur accumulators, AccumulatedSCHessian.cpp:38-39) -- float accumulators, tolerances of tests/test_oracle_marg.py --; and the
    prior update HM += 0.25 (M - Msc), bM += 0.25 (Mb - Mbsc), elementwise fp64 with an exact factor: bit-exact"""
    H, b, mp, col = dense; N = len(bM0)
    scale = np.abs(H[:N, :N]).max(); bscale = np.abs(b[:N]).max()
    assert np.allclose(m["M"], H[:N, :N], rtol=1e-4, atol=1e-5 * scale), (what, "M")
    assert np.allclose(m["Mb"], b[:N], rtol=1e-4, atol=1e-5 * bscale), (what, "Mb")
    S = np.zeros((N, N)); Sb = np.zeros(N)
    for p in mp:
        if win["isFromSensor"][p]:
            continue
        c = col[int(p)]; S += np.outer(H[:N, c], H[:N, c]) / H[c, c]; Sb += H[:N, c] * b[c] / H[c, c]
    assert np.allclose(m["Msc"], S, rtol=1e-3, atol=1e-5 * scale), (what, "Msc")
    assert np.allclose(m["Mbsc"], Sb, rtol=1e-3, atol=1e-5 * bscale + 1e-6), (what, "Mbsc")
    assert np.array_equal(HM1, HM0 + MARG_WEIGHT * (m["M"] - m["Msc"])), (what, "HM")
    assert np.array_equal(bM1, bM0 + MARG_WEIGHT * (m["Mb"] - m["Mbsc"])), (what, "bM")


def marginalize_frame(HM, bM, idx, frameID, state):
    """marginalizeFrame (EnergyFunctional.cpp:434-512) as a Schur complement of the frame's six rows, with FrameHessian::getPrior of frameID 0 (1e10 translation,
    1e11 rotation) and delta_prior = state[:6] (EnergyFunctionalStructs.cpp:28-35).  test_oracle_marg.py::test_marginalize_frame_is_a_schur_complement for any window."""
    N = len(bM); drop = list(range(4 + 6 * idx, 10 + 6 * idx)); keep = [i for i in range(N) if i not in drop]
    prior = np.zeros(6)
    if frameID == 0:
        prior[:3] = TRANS_PRIOR; prior[3:] = ROT_PRIOR
    Dm = HM[np.ix_(drop, drop)] + np.diag(prior); B = HM[np.ix_(keep, drop)]
    H = HM[np.ix_(keep, keep)] - B @ np.linalg.solve(Dm, B.T)
    b = bM[keep] - B @ np.linalg.solve(Dm, bM[drop] + prior * np.asarray(state, np.float64)[:6])
    return 0.5 * (H + H.T), b


def check_marginalized_frame(H2, b2, HM, bM, idx, frameID, state, what=""):
    """the prior after marginalizeFrame against marginalize_frame(), at the tolerances of test_marginalize_frame_is_a_schur_complement (the 6x6 block is inverted,
    so the error follows its condition, not a summation bound)"""
    ref, refb = marginalize_frame(HM, bM, idx, frameID, state)
    assert H2.shape == ref.shape and np.array_equal(H2, H2.T), what
    sc = np.abs(ref).max()
    assert np.allclose(H2, ref, rtol=1e-7, atol=1e-9 * sc), (what, "HM", np.abs(H2 - ref).max(), sc)
    assert np.allclose(b2, refb, rtol=1e-5, atol=1e-7 * (1 + np.abs(refb).max())), (what, "bM", np.abs(b2 - refb).max())
