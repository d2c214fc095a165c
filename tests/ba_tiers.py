"""Back-end windows whose float accumulators cross the 1000-update tier (MatrixAccumulators.h: shiftUp folds a partial into the next tier once its counter
passes 1000), for the reference pin (test_ref_pin_ba_tiers.py), the float64 checks (test_ba_acc_fp64_cpu.py) and the device (test_gpu_ba_tiers.py).

Every window is a subset of one synth.make_ba_window at the KITTI size, with points dropped so that the counts that drive the tiers land exactly on their
targets.  A residual's activity after reset_oob + linearizeAll(False) + applyRes depends only on its own point, the poses and the window's frameEnergyTH
(an input), so it is the same in every subset; the counts are read back from the oracle after the trim and asserted by count_updates().

    top1000 / top1001 / top1002 / top2003   two keyframes; pair (0 -> 1) has exactly that many active residuals (AccumulatorApprox, one per pair), with OOB and
                                            outlier residuals and LiDAR points interleaved (LiDAR residuals count here)
    schur                                   four keyframes; host 1 has exactly 1001 vision points active towards both keyframes 0 and 2 (accD(1,0,2)) and
                                            more active towards 0 only, so accE(1,0) / accEB(1,0) cross at another update; LiDAR points and vision points
                                            without an active residual (ngood == 0) are interleaved and must not count
    hcc                                     two keyframes; exactly 1001 vision points with an active residual (accHcc / accbc, one per window), LiDAR points
                                            and ngood == 0 points interleaved
The schur window is also the marginalisation window: marg_selection() flags host 1's points, all of its counted vision points reach PS_MARGINALIZE, so
marginalizePointsF's accumulators (mode 2) cross 1000 in pair (1 -> 0) and in accD(1,0,2).
numIn1k counts updates, not chunks, so it passes 1000 in the same shiftUp as numIn1: from update 1001 on the completed chunks sit in the 1M partial, and these
windows exercise both shifts.  A 1k partial that holds a sum past a shiftUp would need a counter that counts chunks; nothing here (or in the reference) does."""
import functools
import numpy as np

SEQ = (7, 2000)                        # cached_sequence(7, 2000, KITTI_K, KITTI_WH): the sequence of test_ref_pin_ba.py's KITTI-size pin
LEVELS = 4                             # pyramid levels at 1200 x 360 (the back end reads level 0 only)
TOP_TARGETS = (1000, 1001, 1002, 2003)
SCHUR_HOST, SCHUR_T1, SCHUR_T2 = 1, 0, 2
SCHUR_BOTH = HCC_COUNT = 1001
NAMES = tuple(f"top{n}" for n in TOP_TARGETS) + ("schur", "hcc")
WIN_ARGS = dict(seed=11, sensor_frac=0.4, pose_noise=(0.005, 0.0003), match_noise=0.1, prior_scale=1e-3)


def sequence():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import synth
    from conftest import cached_sequence
    return cached_sequence(SEQ[0], SEQ[1], synth.KITTI_K, synth.KITTI_WH)


def subset(win, keep):
    """the window with only the points where keep is set (and their residuals), in the original order"""
    keep = np.asarray(keep, bool); rb = np.asarray(win["res_begin"]); npt = len(keep)
    rkeep = np.repeat(keep, np.diff(rb))
    out = dict(win)
    for k in ("uv", "idepth", "idepth_zero", "color", "weights", "host", "hasDepthPrior", "isFromSensor"):
        out[k] = np.asarray(win[k])[keep]
    for k in ("r_host", "r_target", "r_hasMatcher", "r_matcher", "r_isNew"):
        out[k] = np.asarray(win[k])[rkeep]
    newidx = np.cumsum(keep) - 1
    out["r_point"] = newidx[np.asarray(win["r_point"])[rkeep]].astype(np.int32)
    out["res_begin"] = np.concatenate([[0], np.cumsum(np.diff(rb)[keep])]).astype(np.int32)
    assert len(out["uv"]) == keep.sum() and npt == len(win["uv"])
    return out


def linearized(win, frames):
    """orc.BAWindow after reset_oob + linearizeAll(False) + applyRes: the state accumulate() and solveSystem() see"""
    import orc
    ob = orc.BAWindow(win, frames); ob.reset_oob(); ob.linearizeAll(False); ob.applyRes()
    return ob


def point_activity(win, active):
    """(nP, nF) bool: point p has an active residual towards frame t"""
    A = np.zeros((len(win["uv"]), int(win["nF"])), bool)
    a = np.asarray(active) != 0
    A[np.asarray(win["r_point"])[a], np.asarray(win["r_target"])[a]] = True
    return A


def count_updates(win, active, status=None):
    """how many updates each float accumulator of accumulate() gets (status given: those of marginalizePointsF, over its PS_MARGINALIZE points):
    top[(h, t)], D[(h, t1, t2)], E[(h, t1)] (accE and accEB alike), hcc (accHcc and accbc alike)"""
    act = np.asarray(active) != 0; rp = np.asarray(win["r_point"])
    if status is not None:
        act = act & (np.asarray(status)[rp] == 2)
    top = {}
    for h, t in zip(np.asarray(win["r_host"])[act], np.asarray(win["r_target"])[act]):
        top[int(h), int(t)] = top.get((int(h), int(t)), 0) + 1
    A = point_activity(win, act); ngood = A.sum(1)
    vis = (ngood > 0) & (np.asarray(win["isFromSensor"]) == 0)
    D, E = {}, {}
    host = np.asarray(win["host"])
    for p in np.where(vis)[0]:
        ts = np.where(A[p])[0]; h = int(host[p])
        for t1 in ts:
            E[h, int(t1)] = E.get((h, int(t1)), 0) + 1
            for t2 in ts:
                D[h, int(t1), int(t2)] = D.get((h, int(t1), int(t2)), 0) + 1
    return dict(top=top, D=D, E=E, hcc=int(vis.sum()))


def _nres(win):
    return np.diff(np.asarray(win["res_begin"]))


def _prefix(mask, n):
    """index just past the n-th set entry of mask"""
    idx = np.where(mask)[0]
    assert len(idx) >= n, (len(idx), n)
    return int(idx[n - 1]) + 1


@functools.lru_cache(maxsize=None)
def _base(nF):
    from sdv_loam_b200 import synth
    seq = sequence()
    win = synth.make_ba_window(seq, list(range(nF)), n_per_frame=4000 if nF == 2 else 6000, **WIN_ARGS)
    import orc
    frames = [orc.Frame(seq.images[k], LEVELS) for k in range(nF)]
    ob = linearized(win, frames); rs = ob.residuals()
    ob.accumulate(); hess = ob.points()["idepth_hessian"]
    return win, frames, rs["active"].copy(), rs["new_state"].copy(), hess


def _others(win, host, n):
    """the first n points of every host other than `host`"""
    keep = np.zeros(len(win["uv"]), bool); hp = np.asarray(win["host"])
    for h in range(int(win["nF"])):
        if h != host:
            keep[np.where(hp == h)[0][:n]] = True
    return keep


@functools.lru_cache(maxsize=None)
def window(name):
    """(window dict, orc frames): one of NAMES"""
    if name.startswith("top"):
        N = int(name[3:]); win, frames, active, _, _ = _base(2)
        host = np.asarray(win["host"]); act0 = point_activity(win, active)[:, 1] & (host == 0)
        keep = _others(win, 0, 60)
        keep[:_prefix(act0, N)] |= host[:_prefix(act0, N)] == 0         # host 0's points up to the N-th active one: the inactive ones in between stay
        return subset(win, keep), frames
    if name == "schur":
        win, frames, active, _, hess = _base(4)
        host = np.asarray(win["host"]); A = point_activity(win, active); vis = np.asarray(win["isFromSensor"]) == 0
        counted = (host == SCHUR_HOST) & vis & A.any(1)
        ok = counted & (_nres(win) >= 3) & (hess > 50)                  # counted points that also reach PS_MARGINALIZE (isInlierNew, setting_minIdepthH_marg)
        both = ok & A[:, SCHUR_T1] & A[:, SCHUR_T2]
        end = _prefix(both, SCHUR_BOTH)
        keep = _others(win, SCHUR_HOST, 40)
        keep[:end] |= (host[:end] == SCHUR_HOST) & (ok[:end] | ~counted[:end])
        return subset(win, keep), frames
    if name == "hcc":
        win, frames, active, _, _ = _base(2)
        host = np.asarray(win["host"]); A = point_activity(win, active); vis = np.asarray(win["isFromSensor"]) == 0
        counted = vis & A.any(1); end = _prefix(counted & (host == 0), HCC_COUNT)
        keep = np.zeros(len(host), bool); keep[:end] = host[:end] == 0
        keep[np.where((host == 1) & ~counted)[0][:60]] = True             # host 1: LiDAR and ngood == 0 points only
        return subset(win, keep), frames
    raise KeyError(name)


def marg_selection(win):
    """the points flagPointsForRemoval is asked to marginalise in the schur window: host 1's points with at least 3 residuals (isInlierNew)"""
    return ((np.asarray(win["host"]) == SCHUR_HOST) & (_nres(win) >= 3)).astype(np.int32)


def check_counts(name, win, active, new_state):
    """the counts the window was built for, exactly; and the interleaved points that must not count are really there"""
    c = count_updates(win, active); host = np.asarray(win["host"]); sensor = np.asarray(win["isFromSensor"]) != 0
    rp = np.asarray(win["r_point"]); act = np.asarray(active) != 0; ngood = np.bincount(rp[act], minlength=len(host))
    if name.startswith("top"):
        pair = (np.asarray(win["r_host"]) == 0) & (np.asarray(win["r_target"]) == 1)
        assert c["top"][0, 1] == int(name[3:]), (name, c["top"][0, 1])
        assert (pair & ~act).sum() > 50 and (pair & act & sensor[rp]).sum() > 300, name          # inactive residuals and LiDAR points interleaved
        assert {1, 2} <= set(np.asarray(new_state)[pair & ~act].tolist()), name                  # both OOB and outliers
    elif name == "schur":
        h, t1, t2 = SCHUR_HOST, SCHUR_T1, SCHUR_T2
        assert c["D"][h, t1, t2] == c["D"][h, t2, t1] == SCHUR_BOTH, (name, c["D"][h, t1, t2])
        assert c["E"][h, t1] == c["D"][h, t1, t1] > SCHUR_BOTH + 50 and c["E"][h, t2] > SCHUR_BOTH, (name, c["E"])
        assert ((host == h) & sensor & (ngood > 0)).sum() > 300 and ((host == h) & ~sensor & (ngood == 0)).sum() > 20, name
    elif name == "hcc":
        assert c["hcc"] == HCC_COUNT, (name, c["hcc"])
        assert (sensor & (ngood > 0)).sum() > 300 and (~sensor & (ngood == 0)).sum() > 20, name
        assert c["E"][0, 1] == HCC_COUNT and c["top"][0, 1] > 1000, (name, c["top"], c["E"])                # one residual per point: accE(0,1) crosses with accHcc
    return c


def check_marg_counts(win, active, status):
    """marginalizePointsF on the schur window: its top accumulator of pair (1 -> 0) and accD(1,0,2) cross 1000"""
    c = count_updates(win, active, status); h, t1, t2 = SCHUR_HOST, SCHUR_T1, SCHUR_T2
    assert c["D"][h, t1, t2] == SCHUR_BOTH and c["top"][h, t1] > 1000 and c["E"][h, t1] > SCHUR_BOTH, c
    return c
