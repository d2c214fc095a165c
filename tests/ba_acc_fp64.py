"""float64 restatement of the back-end's float accumulators (AccumulatedTopHessian / AccumulatedSCHessian with the 1k / 1M tiers of MatrixAccumulators.h) and of
the systems they stitch: HA / bA / Hsc / bsc of accumulate() and M / Mb / Msc / Mbsc of marginalizePointsF, each entry with a bound derived from the actual terms,
for checking the oracle (orc.BAWindow) on the CPU and the device (api.EnergyFunctional) on the GPU with the same code.  The companion of tests/ba_fp64.py (the prior
terms, the assembly and the step): its helpers and constants are used here; its check_marginalized_points compares M / Msc with the empirical tolerances of
tests/test_oracle_marg.py, check_marginalized_points below with the derived bounds (same signature, with dense_marg_system from this module)."""
import math
import numpy as np
from ba_fp64 import MARG_WEIGHT, gamma, stitched_delta

U32 = 2.0 ** -24
F32 = np.float32
CALIB_PRIOR = float(F32(5e9))                          # setting_initialCalibHessian (settings.cpp:27), a float
FRAME0_PRIOR = np.array([float(F32(1e10))] * 3 + [float(F32(1e11))] * 3)   # getPrior of frameID 0: the float settings as doubles (1e11f is 99 999 997 952)
IDEPTH_PRIOR = F32(50 * 50)                            # EFPoint::priorF of a point with a depth prior: setting_idepthFixPrior * SCALE_IDEPTH^2
MARG_PRIOR_FAC = F32(600.0) * F32(600.0)               # setting_idepthFixPriorMargFac (EnergyFunctional.cpp:527)
TIER = 1000                                            # a partial moves up once its counter passes TIER (MatrixAccumulators.h, shiftUp: numIn1 > 1000)


# Every accumulator -- AccumulatorApprox per (host, target) pair (AccumulatedTopHessian.cpp:13-112), AccumulatorXX accD per (host, t1, t2), accE / accEB per (host,
# t1), accHcc / accbc once per window (AccumulatedSCHessian.cpp:10-62) -- adds float32 terms.  They are restated here with the kernels' expression trees (the library
# and the oracle compile with --fmad=false / -ffp-contract=off, so numpy float32 reproduces every term bit for bit) and summed exactly per cell (math.fsum).
#
# Tiers.  update() adds into the running partial A and counts; shiftUp moves A into A1k once the count passes TIER.  numIn1k counts updates too, so it passes
# TIER in the same shiftUp and A1k moves on into A1m at once: from update 1001 on the completed chunks collect in the 1M partial, and the 1k partial is zero after
# every shift.  finish() adds A into A1k and A1k into A1m.  A term therefore passes through at most min(n, TIER + 1) roundings in its chunk, at most
# ceil(n / (TIER + 1)) in the upper partials (entering them, and every later chunk), ceil(n / (TIER + 1)^2) more should a partial ever sit in A1k, and the two of
# finish(): per cell  |float result - exact sum| <= gamma32(tier_depth(n)) * sum |t|  (Higham, section 3.1).  The bound holds for any order of the updates and any
# place of the shift inside update(): a shift after the TopRight / BotRight adds, or a `>= 1000` test, stays inside it.  Only the reference pin sees those
# (tests/test_ref_pin_ba_tiers.py).
# Stitch.  The stitched system is linear in the bucket values: HA = sum over pairs Et^T D Et with Et (10 x N) = [I4 on the calib columns; adHost^T on the host's,
# adTarget^T on the target's], bA = sum Et^T TR; Hsc = sum over (h, t1, t2) Fs(h,t1)^T accD Fs(h,t2) with Fs (6 x N) = [adHost^T, adTarget^T] on the frame columns,
# plus Fs^T accE in the frame-calib blocks, accHcc in the calib block, bsc = sum Fs^T accEB + accbc.  A bucket error delta reaches an entry as |E|^T delta |E|;
# the stitch's own fp64 sums (at most 4 nF^3 + 40 roundings per entry, generously) add gamma(4 nF^3 + 40) * (|E|^T (|D| + delta) |E| + |priors|) per side.
def gamma32(n):
    return n * U32 / (1 - n * U32)


def tier_depth(n):
    """roundings a term of an n-update float accumulator passes through, at most (see above)"""
    c = TIER + 1
    return min(n, c) + -(-n // c) + -(-n // (c * c)) + 2


TRI = [(i, j) for j in range(10) for i in range(j, 10)]                 # AccumulatorApprox Data[] order: cell k = (row i, column j), i >= j
TI, TJ = np.array([i for i, _ in TRI]), np.array([j for _, j in TRI])


def top_terms(J, r):
    """(n, 65) float32 terms of AccumulatorApprox::update(x, y, 1, 0, 1) + the TopRight adds, one row per residual: 55 cells 1*xi*xj + 1*yi*yj + 0*(xi*yj + yi*xj),
    10 cells x_i r0 + y_i r1, with x = [Jpdc[0]; Jpdxi[0]], y = [Jpdc[1]; Jpdxi[1]] of efJ rows (resF 0:2, Jpdxi 2:14, Jpdc 14:22, Jpdd 22:24) and r = resF or res_toZeroF"""
    J = np.asarray(J, F32).reshape(-1, 24); r = np.asarray(r, F32).reshape(-1, 2)
    x = np.concatenate([J[:, 14:18], J[:, 2:8]], 1); y = np.concatenate([J[:, 18:22], J[:, 8:14]], 1)
    with np.errstate(all="ignore"):
        D = ((F32(1) * x[:, TI]) * x[:, TJ] + (F32(1) * y[:, TI]) * y[:, TJ]) + F32(0) * (x[:, TI] * y[:, TJ] + y[:, TI] * x[:, TJ])
        TR = x * r[:, :1] + y * r[:, 1:2]
    return np.concatenate([D, TR], 1).astype(F32)


class Bucket:
    """one float accumulator: its terms in update order (n, cells), exact sum S and sum |t| per cell, and delta = gamma32(tier_depth(n)) * sum |t|.
    lag: cells whose tier shift comes before their add (TopRight / BotRight of AccumulatorApprox::update)"""

    def __init__(self, T, lag=()):
        self.T = np.asarray(T, F32); self.n = n = len(self.T); self.lag = np.zeros(self.T.shape[1], bool); self.lag[list(lag)] = True
        cols = self.T.astype(np.float64).T.tolist()
        self.S = np.array([math.fsum(c) for c in cols]); self.A = np.array([math.fsum(abs(v) for v in c) for c in cols])
        self.delta = gamma32(tier_depth(n)) * self.A

    def open_partial(self):
        """the exact sum of what sits in the running partial A at finish() -- what a finish() that dropped the upper partials would return"""
        k = self.n // (TIER + 1)
        if k == 0:
            return self.S
        T = self.T.astype(np.float64)
        return np.array([math.fsum(T[(TIER + 1) * k - (1 if self.lag[c] else 0):, c].tolist()) for c in range(T.shape[1])])


def _sym10(v):
    M = np.zeros((10, 10)); M[TI, TJ] = v; M[TJ, TI] = v
    return M


def _point_sums(win, J, act, r):
    """per point, in residual order over its active residuals (ba_point_acc_kernel / addPoint): Hdd, bd, Hcd[4] as float32 running sums"""
    rb = np.asarray(win["res_begin"]); nP = len(rb) - 1; J = np.asarray(J, F32); r = np.asarray(r, F32)
    Hdd = np.zeros(nP, F32); bd = np.zeros(nP, F32); Hcd = np.zeros((nP, 4), F32)
    for k in range(int(np.diff(rb).max(initial=0))):
        idx = rb[:-1] + k; ok = idx < rb[1:]; ok[ok] = act[idx[ok]]; i = idx[ok]; j = J[i]
        bd[ok] = bd[ok] + (r[i, 0] * j[:, 22] + r[i, 1] * j[:, 23])
        Hdd[ok] = Hdd[ok] + (j[:, 22] * j[:, 22] + j[:, 23] * j[:, 23])
        Hcd[ok] = Hcd[ok] + (j[:, 14:18] * j[:, 22:23] + j[:, 18:22] * j[:, 23:24])
    return Hdd, bd, Hcd


def _group(keys, order, rows):
    """{key: rows of that key in update order}"""
    out = {}
    if len(rows) == 0:
        return out
    o = np.lexsort((order,) + tuple(np.asarray(keys).T[::-1]))
    keys = [tuple(k) for k in np.asarray(keys)[o].tolist()]; rows = rows[o]
    start = 0
    for i in range(1, len(keys) + 1):
        if i == len(keys) or keys[i] != keys[start]:
            out[keys[start]] = rows[start:i]; start = i
    return out


def normal_equations(win, rs, pts, precalc, frames=None, status=None, res_to_zero=None, variant=None):
    """The float64 restatement of accumulate() -- status None: {"HA", "bA", "Hsc", "bsc"} -- or of marginalizePointsF over its PS_MARGINALIZE points -- status
    given: {"M", "Mb", "Msc", "Mbsc"} --, each as (exact value, bound on |back-end - exact| per entry).  rs: residuals() (efJ, active; new_state and J for the
    variant "inactive"); pts: points() (accumulate() only: HdiF, bdSumF; marginalizePointsF's are restated from efJ with priorF * 600^2); precalc(h, t) -> adHost /
    adTarget; frames: frames() (accumulate() only: the priors of solveSystem's HA / bA).
    variant, restatements of plausible mistakes that the bounds must reject (the exact values change, the bounds stay those of the correct accumulators):
      "inactive"    the top accumulator also counts the inactive residual with the largest Jacobian, with its own last linearisation (J)
      "lidar"       LiDAR points enter the Schur accumulators
      "lost_tiers"  finish() returns only the running partial, losing the completed 1000-update chunks (a no-op for every bucket below the tier)
    Returns (equations, counts) with counts = {"top": {(h, t): n}, "D": {(h, t1, t2): n}, "E": {(h, t1): n}, "hcc": n}: the updates each accumulator got."""
    marg = status is not None
    nF = int(win["nF"]); N = 4 + 6 * nF; rp = np.asarray(win["r_point"]); rh = np.asarray(win["r_host"]); rt = np.asarray(win["r_target"])
    J = np.asarray(rs["efJ"], F32); act = np.asarray(rs["active"]) != 0
    if marg:
        act = act & (np.asarray(status)[rp] == 2)
    r = np.asarray(res_to_zero, F32) if marg else J[:, :2]
    sensor = np.asarray(win["isFromSensor"]) != 0
    # ---- top: one AccumulatorApprox per pair, residuals in order
    ia = np.where(act)[0]; T = top_terms(J[ia], r[ia])
    if variant == "inactive":
        cand = np.where(~(np.asarray(rs["active"]) != 0) & ((np.asarray(status)[rp] == 2) if marg else True))[0]
        Jin = np.asarray(rs["J"], F32)
        k = int(cand[np.argmax(np.abs(Jin[cand]).sum(1))])
        ia = np.append(ia, k); T = np.concatenate([T, top_terms(Jin[k:k + 1], Jin[k:k + 1, :2] if not marg else r[k:k + 1])])
    top = {k: Bucket(v, lag=range(55, 65)) for k, v in _group(np.stack([rh[ia], rt[ia]], 1), ia, T).items()}
    # ---- Schur: per point HdiF / bdSumF / Hcd, then accD / accE+accEB / accHcc+accbc over the counted points
    Hdd, bd, Hcd = _point_sums(win, J, act, r)
    ngood = np.bincount(rp[act], minlength=len(sensor))
    if marg:
        prior = np.where(np.asarray(win["hasDepthPrior"]) != 0, IDEPTH_PRIOR, F32(0)).astype(F32) * MARG_PRIOR_FAC
        Hh = (Hdd + F32(0)) + prior; Hh = np.where(Hh < 1e-10, F32(1e-10), Hh).astype(F32)
        Hdi = (1.0 / Hh.astype(np.float64)).astype(F32); bds = (bd + F32(0)).astype(F32)
    else:
        Hdi = np.asarray(pts["HdiF"], F32); bds = np.asarray(pts["bdSumF"], F32)
    counted = (ngood > 0) & (~sensor if variant != "lidar" else True)
    JJ = np.asarray(rs["JpJdF"], F32)[:, :6] if (not marg and "JpJdF" in rs) else (J[:, 2:8] * J[:, 22:23] + J[:, 8:14] * J[:, 23:24]).astype(F32)
    slots = [[] for _ in range(len(sensor))]
    for i in ia if variant != "inactive" else ia[:-1]:
        slots[rp[i]].append(i)
    K = max((len(s) for s in slots), default=0); R = np.full((len(sensor), max(K, 1)), -1)
    for p, s in enumerate(slots):
        R[p, :len(s)] = s
    host = np.asarray(win["host"]); dk, dord, drow, ek, eord, erow = [], [], [], [], [], []
    for a in range(K):
        Pa = np.where(counted & (R[:, a] >= 0))[0]; r1 = R[Pa, a]; w1 = Hdi[Pa, None] * JJ[r1]
        ek.append(np.stack([host[Pa], rt[r1]], 1)); eord.append(Pa)
        erow.append(np.concatenate([(w1[:, :, None] * Hcd[Pa, None, :]).reshape(-1, 24), (Hdi[Pa] * bds[Pa])[:, None] * JJ[r1]], 1))
        for b in range(K):
            P = np.where(counted & (R[:, a] >= 0) & (R[:, b] >= 0))[0]; r1, r2 = R[P, a], R[P, b]
            dk.append(np.stack([host[P], rt[r1], rt[r2]], 1)); dord.append(P)
            drow.append(((Hdi[P, None] * JJ[r1])[:, :, None] * JJ[r2][:, None, :]).reshape(-1, 36))
    cat = lambda xs, w: np.concatenate(xs) if xs else np.zeros((0, w))
    D = {k: Bucket(v) for k, v in _group(cat(dk, 3).astype(int), cat(dord, 1).ravel() if dord else np.zeros(0), cat(drow, 36).astype(F32)).items()}
    E = {k: Bucket(v) for k, v in _group(cat(ek, 2).astype(int), cat(eord, 1).ravel() if eord else np.zeros(0), cat(erow, 30).astype(F32)).items()}
    Pc = np.where(counted)[0]
    hc = np.concatenate([((Hdi[Pc, None] * Hcd[Pc])[:, :, None] * Hcd[Pc, None, :]).reshape(-1, 16), (bds[Pc] * Hdi[Pc])[:, None] * Hcd[Pc]], 1).astype(F32)
    HC = Bucket(hc) if len(Pc) else None
    # ---- stitch
    val = (lambda B: B.open_partial()) if variant == "lost_tiers" else (lambda B: B.S)
    ads = {}

    def ad(h, t):
        if (h, t) not in ads:
            pc = precalc(h, t); ads[h, t] = (np.asarray(pc["adHost"], np.float64), np.asarray(pc["adTarget"], np.float64))
        return ads[h, t]

    def frame_map(h, t):
        aH, aT = ad(h, t); F = np.zeros((6, N)); F[:, 4 + 6 * h:10 + 6 * h] += aH.T; F[:, 4 + 6 * t:10 + 6 * t] += aT.T
        return F

    H, b, Hd, bd_, Ha, ba = (np.zeros((N, N)), np.zeros(N), np.zeros((N, N)), np.zeros(N), np.zeros((N, N)), np.zeros(N))   # value, bucket error, |.| for gamma
    for (h, t), B in top.items():
        Et = np.zeros((10, N)); Et[:4, :4] = np.eye(4); Et[4:] = frame_map(h, t); Ea = np.abs(Et)
        H += Et.T @ _sym10(val(B)[:55]) @ Et; b += Et.T @ val(B)[55:]
        Hd += Ea.T @ _sym10(B.delta[:55]) @ Ea; bd_ += Ea.T @ B.delta[55:]
        Ha += Ea.T @ _sym10(np.abs(B.S[:55]) + B.delta[:55]) @ Ea; ba += Ea.T @ (np.abs(B.S[55:]) + B.delta[55:])
    Hs, bs, Hsd, bsd, Hsa, bsa = (np.zeros((N, N)), np.zeros(N), np.zeros((N, N)), np.zeros(N), np.zeros((N, N)), np.zeros(N))
    for (h, t1, t2), B in D.items():
        F1, F2 = frame_map(h, t1), frame_map(h, t2)
        Hs += F1.T @ val(B).reshape(6, 6) @ F2; Hsd += np.abs(F1).T @ B.delta.reshape(6, 6) @ np.abs(F2)
        Hsa += np.abs(F1).T @ (np.abs(B.S) + B.delta).reshape(6, 6) @ np.abs(F2)
    for (h, t1), B in E.items():
        F1 = frame_map(h, t1); Fa = np.abs(F1)
        for M, v in ((Hs, F1.T @ val(B)[:24].reshape(6, 4)), (Hsd, Fa.T @ B.delta[:24].reshape(6, 4)), (Hsa, Fa.T @ (np.abs(B.S) + B.delta)[:24].reshape(6, 4))):
            M[:, :4] += v; M[:4, :] += v.T
        bs += F1.T @ val(B)[24:]; bsd += Fa.T @ B.delta[24:]; bsa += Fa.T @ (np.abs(B.S) + B.delta)[24:]
    if HC is not None:
        Hs[:4, :4] += val(HC)[:16].reshape(4, 4); Hsd[:4, :4] += HC.delta[:16].reshape(4, 4); Hsa[:4, :4] += (np.abs(HC.S) + HC.delta)[:16].reshape(4, 4)
        bs[:4] += val(HC)[16:]; bsd[:4] += HC.delta[16:]; bsa[:4] += (np.abs(HC.S) + HC.delta)[16:]
    if not marg:                                                       # accumulateAF_MT's priors (usePrior / useDelta): calib, frameID 0
        st = np.asarray(frames["state"], np.float64); cD = stitched_delta(win, frames)[:4]
        pr = np.concatenate([[CALIB_PRIOR] * 4] + [FRAME0_PRIOR if int(win["frameID"][f]) == 0 else np.zeros(6) for f in range(nF)])
        pb = pr * np.concatenate([cD, st[:, :6].reshape(-1)])
        H[np.diag_indices(N)] += pr; b += pb; Ha[np.diag_indices(N)] += pr; ba += np.abs(pb)
    g = 2 * gamma(4 * nF ** 3 + 40)
    names = ("M", "Mb", "Msc", "Mbsc") if marg else ("HA", "bA", "Hsc", "bsc")
    eq = dict(zip(names, ((H, Hd + g * Ha), (b, bd_ + g * ba), (Hs, Hsd + g * Hsa), (bs, bsd + g * bsa))))
    counts = dict(top={k: B.n for k, B in top.items()}, D={k: B.n for k, B in D.items()}, E={k: B.n for k, B in E.items()}, hcc=HC.n if HC is not None else 0)
    return eq, counts


def check_equations(eq, got, what="", rep=None):
    """every entry of the back-end's HA / bA / Hsc / bsc (or M / Mb / Msc / Mbsc) within its bound of the exact value; eq: normal_equations()[0] (or the pair);
    rep: a tracker_fp64.Report that keeps the worst error / bound per check"""
    if isinstance(eq, tuple):
        eq = eq[0]
    for name, (ref, bnd) in eq.items():
        err = np.abs(np.asarray(got[name], np.float64) - ref); k = int(np.argmax(err - bnd))
        assert np.all(err <= bnd), (what, name, np.unravel_index(k, err.shape), float(err.flat[k]), float(bnd.flat[k]))
        if rep is not None:
            rep.check(name, float(np.max(np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1), 0))), 1.0)


def rejected(eq, variant, got):
    """the names of the quantities in which some entry of the back-end's `got` lies outside the correct bounds (eq) around a variant's exact values: a back-end
    that computed the variant would have been caught there"""
    eq, variant = (e[0] if isinstance(e, tuple) else e for e in (eq, variant))
    return [name for name, (_, bnd) in eq.items() if np.any(np.abs(np.asarray(got[name], np.float64) - variant[name][0]) > bnd)]


def dense_marg_system(win, efJ, res_to_zero, active, precalc, status):
    """the float64 restatement of marginalizePointsF's accumulators (normal_equations(mode=2)) over the PS_MARGINALIZE points, from efJ / res_toZeroF / activity /
    status as either back-end returns them after flagPointsForRemoval: precalc(h, t) -> dict with adHost / adTarget"""
    return normal_equations(win, dict(efJ=efJ, active=active), None, precalc, status=status, res_to_zero=res_to_zero)


def check_marginalized_points(win, m, HM0, bM0, HM1, bM1, dense, what="", rep=None):
    """marginalizePointsF (EnergyFunctional.cpp:514-576): M / Mb / Msc / Mbsc entry by entry within the tier-aware bounds of normal_equations() (LiDAR points never
    reach the Schur accumulators, AccumulatedSCHessian.cpp:38-39); and the prior update HM += 0.25 (M - Msc), bM += 0.25 (Mb - Mbsc), elementwise fp64 with an
    exact factor: bit-exact"""
    check_equations(dense, m, what, rep)
    assert np.array_equal(HM1, HM0 + MARG_WEIGHT * (m["M"] - m["Msc"])), (what, "HM")
    assert np.array_equal(bM1, bM0 + MARG_WEIGHT * (m["Mb"] - m["Mbsc"])), (what, "bM")
