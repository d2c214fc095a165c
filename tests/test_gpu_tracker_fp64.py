"""GPU tracker kernels against the float64 reference (tests/tracker_fp64.py), with derived error bounds instead of empirical tolerances.

  a. coarse_res_gs_kernel (step-wise calcRes + calcGSSSE) on the KITTI, KITTI-360 and S-STRESS clouds: nE / nSat exact, E, H, b and the flow
     indicators within bound(m), m = points per thread of the launch;
  b. clouds shaped for the edges: point counts around the block size and the grid cap, 1/64-px and one-ulp lattices across the image-bound
     checks, residuals exactly at huberTH / cutoffTH, NaN and +-inf under a bilinear tap versus only under a central-difference tap;
  c. track_cluster_kernel (the device-resident LM) at every point-count edge of every launch configuration: lastResiduals and flow at the
     returned pose against the reference, single jobs against batched ones, one pyramid level at a time, the empty-level path;
  d. the real-data tracks of KITTI, KITTI-360 and S-STRESS in both configurations, lastResiduals and flow at the returned pose.
Every test prints its worst error as a fraction of its bound."""
import numpy as np
import pytest
import orc
import tracker_fp64 as tf
from conftest import cached_sequence

pytestmark = pytest.mark.gpu
ID7 = np.array([1, 0, 0, 0, 0, 0, 0.0])
F = np.float32
CFGS = [(64, 1), (128, 1), (256, 1), (128, 2), (128, 4), (256, 8), (256, 16)]


def _api():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _p4(synth, seq, n):
    pts = synth.select_points(seq.images[0], seq.clouds[0], n)
    return np.concatenate([pts, np.full((len(pts), 1), 1e-3, F)], 1).astype(F)


def _tgt(synth, seq):
    return orc.se3_from_rt(*synth.rel_pose(seq.R[0], seq.t[0], seq.R[1], seq.t[1]))


def _kitti(kitti_seq, n_slots=1, **ctxkw):
    """KITTI frames 0 / 1 on the GPU and in the oracle, and the real reference clouds of frame 0 on every level."""
    api, synth = _api(); w, h = synth.KITTI_WH; L = 4
    ctx = api.Context(synth.KITTI_K, w, h, max_frames=8, n_tracker_slots=n_slots, **ctxkw)
    ctx.makeImages(0, kitti_seq.images[0]); ctx.makeImages(1, kitti_seq.images[1])
    f0, f1 = orc.Frame(kitti_seq.images[0], L), orc.Frame(kitti_seq.images[1], L)
    o = orc.CoarseTracker(w, h, L, synth.KITTI_K); p4 = _p4(synth, kitti_seq, 2000); o.setCoarseTrackingRef(f0, p4, np.zeros(len(p4), np.int32))
    clouds = [o.cloud(l) for l in range(L)]
    return api, synth, ctx, f0, f1, clouds


def _rep_cloud(c, n, seed=0):
    """n points: the real cloud repeated, every copy after the first jittered by the same sub-pixel float32 offsets on both sides."""
    k = len(c[0]); idx = (np.arange(n) + k // 2) % k                         # start mid-cloud: the first points are well inside the image
    d = np.random.default_rng(seed).uniform(-0.25, 0.25, (n, 2)).astype(F); d[:min(n, k)] = 0
    return [F(c[0][idx]) + d[:, 0], F(c[1][idx]) + d[:, 1], c[2][idx].copy(), c[3][idx].copy()]


def _set_both(tr, otr, f0, lvl, cl, ref_a=0.0, ref_b=0.0):
    tr.setCloud(0, lvl, *cl, ref_a, ref_b); otr.setCloud(f0, lvl, *cl, ref_a, ref_b)


def _step_check(tr, otr, frame_id, frame, lvl, T, a, b, cutoff, rep, tag, sms, ref_b=0.0, gs=True):
    n = len(otr.cloud(lvl)[0]); m = tf.m_step(n, sms)
    ref = tf.Ref(otr, frame, lvl, T, a, b, cutoff, ref_b=ref_b, gs=gs)
    rs = tr.calcRes(frame_id, lvl, T, a, b, cutoff)
    ref.check_res(rs, m, rep, tag)
    if gs and n > 0:
        H, bb = tr.calcGSSSE(lvl); ref.check_gs(H, bb, m, rep, tag)
    return ref, rs


# ------------------------------------------------------------------------------------------------ a. step-wise kernel on real clouds
@pytest.mark.parametrize("size", ["kitti", "kitti360", "stress"])
def test_stepwise_vs_reference(kitti_seq, size):
    api, synth = _api(); sms = _sms(); rep = tf.Report(f"step-wise {size}")
    if size == "kitti":
        w, h = synth.KITTI_WH; L = 4; K = synth.KITTI_K; seq = kitti_seq; p4 = _p4(synth, seq, 2000)
        ctx = api.Context(K, w, h, max_frames=4); ctx.makeImages(0, seq.images[0]); ctx.makeImages(1, seq.images[1])
        tr = api.CoarseTracker(ctx, 0); tr.setCoarseTrackingRef(0, p4, np.zeros(len(p4), np.int32), 0.0, 1.0)
        otr = orc.CoarseTracker(w, h, L, K); otr.setCoarseTrackingRef(orc.Frame(seq.images[0], L), p4, np.zeros(len(p4), np.int32), 0.0, 1.0)
        f1 = orc.Frame(seq.images[1], L)
    else:
        from test_gpu_sizes import _seq, _tracker_pair
        S, seq = _seq(size); ctx, tr, otr, f1, L, _ = _tracker_pair(api, synth, S, seq)
    Tgt = _tgt(synth, seq); ms = []
    for T in (ID7, orc.se3_mul(orc.se3_exp([0.01, 0.0, 0.02, 1e-3, -1e-3, 5e-4]), Tgt)):
        for l in range(L):
            ms.append((l, len(otr.cloud(l)[0]), tf.m_step(len(otr.cloud(l)[0]), sms)))
            for cutoff, (a, b) in ((20.0, (0.0, 0.0)), (40.0, (0.03, -2.0))):
                _step_check(tr, otr, 1, f1, l, T, a, b, cutoff, rep, f"L{l}", sms, ref_b=1.0)
    rep.print(); print("  (level, n, m):", sorted(set(ms)))
    ctx.close()


# ------------------------------------------------------------------------------------------------ b. clouds shaped for the edges
def test_stepwise_point_counts(kitti_seq):
    """n around the block size and at the grid cap 4 SMs x 256, where each thread starts taking a second point."""
    sms = _sms(); api, synth, ctx, f0, f1, clouds = _kitti(kitti_seq); rep = tf.Report("step-wise point counts")
    w, h = synth.KITTI_WH; tr = api.CoarseTracker(ctx, 0); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
    cap = 4 * sms * 256; T = orc.se3_mul(orc.se3_exp([0.01, 0.0, 0.02, 1e-3, -1e-3, 5e-4]), _tgt(synth, kitti_seq))
    assert tf.m_step(cap, sms) == 1 and tf.m_step(cap + 1, sms) == 2
    for n in (0, 1, 31, 32, 33, 255, 256, 257, cap, cap + 1):
        _set_both(tr, otr, f0, 0, _rep_cloud(clouds[0], n, seed=n))
        for cutoff, (a, b) in ((20.0, (0.0, 0.0)), (40.0, (0.03, -2.0))):
            _step_check(tr, otr, 1, f1, 0, T, a, b, cutoff, rep, f"n={n}" if n < 300 else "n=cap" + ("+1" if n > cap else ""), sms)
    rep.print(); ctx.close()


def _ulp_window(x0, k):
    b = np.array([x0], F).view(np.int32)[0]
    return np.arange(b - k, b + k + 1, dtype=np.int32).view(F)


def _project_identity(Ki, K4, x, y):
    """Ku, Kv of stage_project / eval_point at the identity pose (RKi = Ki exactly, t = 0)."""
    Ki = np.asarray(Ki, F); one = F(1); z = F(0)
    p = [((Ki[i, 0] * x + Ki[i, 1] * y) + Ki[i, 2] * one) + z for i in range(3)]
    return F(K4[0]) * (p[0] / p[2]) + F(K4[2]), F(K4[1]) * (p[1] / p[2]) + F(K4[3])


def _lattice(otr, w, h):
    """1/64-px lattices and 1-ulp windows straddling Ku = 2, Ku = w-3, Kv = 2, Kv = h-3 at the identity, with positive, zero and negative idepth."""
    Ki, K4 = otr.Ki(0), otr.K(0); xs, ys, hits = [], [], {}
    ym, xm = F(h / 2 + 0.37), F(w / 2 + 0.41)
    for name, b0, along_x in (("Ku=2", 2.0, True), ("Ku=w-3", w - 3.0, True), ("Kv=2", 2.0, False), ("Kv=h-3", h - 3.0, False)):
        win = _ulp_window(F(b0), 3000)
        cand = np.concatenate([win, F(b0) + np.arange(-64, 65, dtype=F) / F(64)]).astype(F)
        px, py = (cand, np.full(len(cand), ym, F)) if along_x else (np.full(len(cand), xm, F), cand)
        Ku, Kv = _project_identity(Ki, K4, px, py); K = Ku if along_x else Kv
        on = K == F(b0)
        hits[name] = int(on.sum())
        near = np.abs(K.astype(np.float64) - b0) < 1e-3                       # the exact hits and their one-ulp neighbours in K
        keep = np.concatenate([np.flatnonzero(on)[:32], np.flatnonzero(near & ~on)[:32], np.arange(len(win), len(cand))])
        xs.append(px[keep]); ys.append(py[keep])
    gx, gy = np.meshgrid(np.arange(-2, 3, dtype=F) * F(7.25), np.arange(-2, 3, dtype=F) * F(5.5))   # a few points mid-image, in front at every pose
    xs.append(xm + gx.reshape(-1)); ys.append(ym + gy.reshape(-1))
    idv = np.array([0.05, 0.2, 0.0, -0.05, 1.0], F)                        # every lattice point with every idepth
    x, y = np.repeat(np.concatenate(xs), len(idv)), np.repeat(np.concatenate(ys), len(idv)); n = len(x)
    idp = np.tile(idv, n // len(idv))
    col = (F(60) + F(40) * np.sin(np.arange(n, dtype=F))).astype(F)
    return [x, y, idp, col], hits


def test_bounds_lattice(kitti_seq):
    """Points exactly on the image-bound checks (and one ulp either side), idepth <= 0 and points behind the camera: counts exactly as the
    oracle, sums within the bound; then the LM kernel on the same lattice against a constant target, where the pose cannot move off the
    identity and every evaluation sees the boundary points exactly on the boundary."""
    sms = _sms(); api, synth, ctx, f0, f1, _ = _kitti(kitti_seq); rep = tf.Report("bounds lattice")
    w, h = synth.KITTI_WH; tr = api.CoarseTracker(ctx, 0); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
    cl, hits = _lattice(otr, w, h)
    print("\n  lattice points exactly on each bound:", hits)
    assert all(v > 0 for v in hits.values()), hits
    _set_both(tr, otr, f0, 0, cl)
    behind = orc.se3_exp([0.0, 0.0, -8.0, 0.0, 0.0, 0.0])                   # pt2 = 1 - 8 idepth: the idepth 0.2 / 1.0 points are behind the camera
    for T in (ID7, behind):
        ref, rs = _step_check(tr, otr, 1, f1, 0, T, 0.0, 0.0, 20.0, rep, "step", sms)
        assert 0 < ref.nE < len(cl[0])
    # LM on a constant image: zero gradients, so the pose rows of H are zero, the step leaves the pose at the identity and only a, b move
    const = np.full((h, w), 90.0, F); ctx.makeImages(4, const); f4 = orc.Frame(const, 4)
    rg = tr.trackNewestCoarse(4, ID7, (0.0, 0.0), coarsest=0); ro = otr.trackNewestCoarse(f4, ID7, (0.0, 0.0), 0)
    assert np.array_equal(rg["T"], ID7) and np.array_equal(ro["T"], ID7)
    assert np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"]) and np.array_equal(rg["evals"], ro["evals"])
    ref = tf.Ref(otr, f4, 0, rg["T"], *rg["ab"], 20.0, gs=False)
    assert rg["evals"][0] == len(cl[0]) * (rg["iterations"][0] + 1)
    rep.check("LM lastRes", abs(rg["lastResiduals"][0] - ref.lastRes), ref.lastres_bound(tf.m_lm(len(cl[0]), 128, 1)))
    rep.print(); ctx.close()


def test_exact_thresholds(kitti_seq):
    """A patch of zeros in the target: hit0 = 0 exactly, so at a = b = 0 the residual is exactly -color.  Colours at +-huberTH, +-cutoffTH and
    their float neighbours put |r| < huber and |r| > cutoff on the boundary itself."""
    sms = _sms(); api, synth, ctx, f0, f1, _ = _kitti(kitti_seq); rep = tf.Report("exact thresholds")
    w, h = synth.KITTI_WH; tr = api.CoarseTracker(ctx, 0); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
    img = kitti_seq.images[1].astype(F).copy(); img[100:200, 400:800] = 0; ctx.makeImages(2, img); f2 = orc.Frame(img, 4)
    vals = []
    for base in (6.0, 20.0, 40.0):
        for s in (1, -1):
            vals += [s * np.nextafter(F(base), F(0)), s * F(base), s * np.nextafter(F(base), F(1e9))]
    vals = np.array(vals + [0.0, 3.0, -10.0, 30.0], F); k = len(vals)
    gx, gy = np.meshgrid(np.arange(410, 790, 6), np.arange(108, 192, 6))
    x = (gx.reshape(-1) + 0.5).astype(F); y = (gy.reshape(-1) + 0.25).astype(F); n = len(x)
    cl = [x, y, np.full(n, 0.1, F), np.tile(vals, n // k + 1)[:n]]
    _set_both(tr, otr, f0, 0, cl)
    for cutoff in (20.0, 40.0):
        ref, rs = _step_check(tr, otr, 2, f2, 0, ID7, 0.0, 0.0, cutoff, rep, f"cutoff {cutoff:g}", sms)
        res = otr.warped()[5][:ref.nW]
        assert ref.nE == n and np.any(np.abs(res) == F(cutoff)) and np.any(np.abs(res) == F(6.0))      # on the boundary, not saturated
        assert ref.nSat == int((np.abs(cl[3]) > F(cutoff)).sum())
    rep.print(); ctx.close()


def test_nonfinite_pixels(kitti_seq):
    """NaN / +inf / -inf in the target: under a bilinear tap the point is skipped; only under a central-difference tap the gradient is zeroed
    and the point counts."""
    sms = _sms(); api, synth, ctx, f0, f1, _ = _kitti(kitti_seq); rep = tf.Report("non-finite pixels")
    w, h = synth.KITTI_WH; tr = api.CoarseTracker(ctx, 0); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
    img = kitti_seq.images[1].astype(F).copy(); bad = [(600, 150, np.nan), (700, 200, np.inf), (800, 250, -np.inf)]
    for px, py, val in bad:
        img[py, px] = val
    ctx.makeImages(3, img); f3 = orc.Frame(img, 4)
    bil = [(-0.5, -0.5), (0.25, 0.25), (-0.75, 0.25), (0.25, -0.75)]          # the bad pixel is one of the 2x2 bilinear taps
    cen = [(0.25, 1.25), (-0.75, 1.25), (1.25, 0.25), (-1.75, 0.25), (1.25, -0.75), (-1.75, -0.75), (0.25, -1.75), (-0.75, -1.75)]   # only a gradient tap
    pts = [(px + dx, py + dy) for px, py, _ in bad for dx, dy in bil + cen]
    x = np.array([p[0] for p in pts], F); y = np.array([p[1] for p in pts], F); n = len(x)
    cl = [x, y, np.full(n, 0.1, F), np.full(n, 50.0, F)]
    _set_both(tr, otr, f0, 0, cl)
    ref, rs = _step_check(tr, otr, 3, f3, 0, ID7, 0.0, 0.0, 1e4, rep, "identity", sms)
    assert ref.nE == len(bad) * len(cen), ref.nE
    wp = otr.warped()[:, :ref.nW]; assert np.all(np.isfinite(wp))
    rep.print(); ctx.close()


# ------------------------------------------------------------------------------------------------ c. the LM sweep at every point-count edge
def _lm_sizes(threads, cluster, cap):
    S = threads * cluster
    ns = {1, 31, 33, threads - 1, threads + 1, S - 1, S + 1, 4 * S - 1, 4 * S, 4 * S + 1, 8 * S + 1, 12 * S - 1, 12 * S + threads + 1}
    return sorted(n for n in ns if 0 < n <= cap)


def _lm_check(rg, otr, f1, lvl, n, m, rep, tag):
    """lastResiduals[lvl] and (level 0) flow[0] / flow[2] at the returned (T, ab) against the reference."""
    its = int(rg["iterations"][lvl])
    reps = int(rg["evals"][lvl] // n) - (its + 1)                          # cutoff repeats at level entry, each doubles the cutoff
    assert rg["evals"][lvl] == n * (its + 1 + reps) and 0 <= reps <= (2 if n < 64 else 0), (tag, rg["evals"], rg["iterations"])
    ref = tf.Ref(otr, f1, lvl, rg["T"], *rg["ab"], 20.0 * 2 ** reps, gs=False)
    assert ref.nE > 0, (tag, "every point left the image")
    rep.check("lastRes", abs(rg["lastResiduals"][lvl] - ref.lastRes), ref.lastres_bound(m))
    if lvl == 0:
        fN = float(F(ref.n_flow)) + 0.1
        rep.check("flow[0]", abs(rg["flow"][0] - ref.rs[2]), ref.sum_bound(tf.IDX_FT, m) / fN)
        rep.check("flow[2]", abs(rg["flow"][2] - ref.rs[4]), ref.sum_bound(tf.IDX_FRT, m) / fN)
    return ref


@pytest.mark.parametrize("cfg", CFGS)
def test_lm_point_count_edges(kitti_seq, cfg):
    threads, cluster = cfg; sms = _sms(); rep = tf.Report(f"LM sweep {threads}x{cluster}")
    api, synth = _api(); w, h = synth.KITTI_WH
    ns = _lm_sizes(threads, cluster, w * h)
    api, synth, ctx, f0, f1, clouds = _kitti(kitti_seq, n_slots=len(ns), track_threads=threads, cluster_size=cluster)
    T0 = orc.se3_mul(orc.se3_exp([0.02, -0.01, 0.03, 1e-3, -1e-3, 5e-4]), _tgt(synth, kitti_seq)); ab0 = (0.0, 0.0)
    singles, oracles, worst_pose = [], [], 0.0
    for i, n in enumerate(ns):
        tr = api.CoarseTracker(ctx, i); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
        _set_both(tr, otr, f0, 0, _rep_cloud(clouds[0], n, seed=n))
        rg = tr.trackNewestCoarse(1, T0, ab0, coarsest=0); singles.append(rg); oracles.append(otr)
        _lm_check(rg, otr, f1, 0, n, tf.m_lm(n, threads, cluster), rep, n)
        # the step-wise kernel at the same pose: the same E / nE within both kernels' bounds
        _step_check(tr, otr, 1, f1, 0, rg["T"], *rg["ab"], 20.0, rep, "step-wise", sms, gs=False)
        if n <= 20000:
            ro = otr.trackNewestCoarse(f1, T0, ab0, 0)
            same = np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"])
            if n < 64 and not same:                                        # a few dozen points: the step-norm stop (|inc| > 1e-3) can flip on the last float bit
                print(f"  n={n}: LM path differs from the oracle's (iterations {rg['iterations'][0]} vs {ro['iterations'][0]})"); continue
            assert np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"]), (n, rg["iterations"], ro["iterations"])
            assert np.array_equal(rg["evals"], ro["evals"]), (n, rg["evals"], ro["evals"])
            # same path, sums in another order: 1e-5 on real-size clouds; a few hundred points condition the last step less well
            dp = np.abs(orc.se3_log(orc.se3_mul(rg["T"], orc.se3_inv(ro["T"])))).max(); worst_pose = max(worst_pose, dp)
            assert dp < (1e-5 if n >= 1000 else 1e-4) and rg["good"] == ro["good"], (n, dp)
    # every size as its own job on its own slot, in one launch: bit-identical to the single-job runs
    T = np.tile(T0, (len(ns), 1)); ab = np.tile(np.array(ab0), (len(ns), 1))
    rb = ctx.trackBatch(list(range(len(ns))), [1] * len(ns), T, ab, coarsest=0)
    for i, rg in enumerate(singles):
        assert np.array_equal(T[i], rg["T"]) and np.array_equal(ab[i], rg["ab"]), ns[i]
        assert np.array_equal(rb["lastResiduals"][i], rg["lastResiduals"], equal_nan=True) and np.array_equal(rb["flow"][i], rg["flow"])
        assert np.array_equal(rb["iterations"][i], rg["iterations"]) and np.array_equal(rb["evals"][i], rg["evals"])
    rep.print(); print("  sizes:", ns, f"worst pose difference to the oracle's LM {worst_pose:.1e}"); ctx.close()


@pytest.mark.parametrize("cfg", [(128, 1), (256, 16)])
def test_lm_one_level_at_a_time(kitti_seq, cfg):
    """Empty levels first (nE = 0: NaN H, zeroed step, one rejected iteration, NaN lastResiduals, unchanged pose) against the oracle's LM; then
    a cloud on level l only, starting at coarsest = l with the finer levels empty, checked through lastResiduals[l]."""
    threads, cluster = cfg; rep = tf.Report(f"LM per level {threads}x{cluster}")
    api, synth, ctx, f0, f1, clouds = _kitti(kitti_seq, n_slots=4, track_threads=threads, cluster_size=cluster)
    w, h = synth.KITTI_WH; T0 = orc.se3_mul(orc.se3_exp([0.02, -0.01, 0.03, 1e-3, -1e-3, 5e-4]), _tgt(synth, kitti_seq))
    tr = api.CoarseTracker(ctx, 0); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
    _set_both(tr, otr, f0, 0, [np.zeros(0, F)] * 4)
    rg = tr.trackNewestCoarse(1, T0, (0.0, 0.0), coarsest=3); ro = otr.trackNewestCoarse(f1, T0, (0.0, 0.0), 3)
    assert np.array_equal(rg["iterations"][:4], [1, 1, 1, 1]) and np.array_equal(rg["accepts"][:4], [0, 0, 0, 0])
    assert np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"])
    assert np.array_equal(np.isnan(rg["lastResiduals"]), np.isnan(ro["lastResiduals"])) and np.all(np.isnan(rg["lastResiduals"][:4]))
    assert np.array_equal(rg["T"], T0) and np.array_equal(ro["T"], T0)
    for l in (1, 2, 3):
        tr = api.CoarseTracker(ctx, l); otr = orc.CoarseTracker(w, h, 4, synth.KITTI_K)
        _set_both(tr, otr, f0, l, clouds[l]); n = len(clouds[l][0])
        rg = tr.trackNewestCoarse(1, T0, (0.0, 0.0), coarsest=l); ro = otr.trackNewestCoarse(f1, T0, (0.0, 0.0), l)
        _lm_check(rg, otr, f1, l, n, tf.m_lm(n, threads, cluster), rep, l)
        assert np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"])
        assert np.abs(orc.se3_log(orc.se3_mul(rg["T"], orc.se3_inv(ro["T"])))).max() < 1e-5
        assert np.all(np.isnan(rg["lastResiduals"][:l])) and np.array_equal(rg["iterations"][:l], [1] * l)
    rep.print(); ctx.close()


# ------------------------------------------------------------------------------------------------ d. real-data tracks, held tighter
@pytest.mark.parametrize("cfg", [(128, 1), (256, 16)])
@pytest.mark.parametrize("size", ["kitti", "kitti360", "stress"])
def test_real_track_vs_reference(kitti_seq, size, cfg):
    """trackNewestCoarse on the real clouds: lastResiduals[0] and the flow indicators at the returned pose against the reference.  At
    (128, 1) the S-STRESS level-0 sweep accumulates 1 280 points per thread in float32 before fp64 takes over; the ratio printed is what
    that costs against its bound."""
    threads, cluster = cfg; api, synth = _api(); rep = tf.Report(f"track {size} {threads}x{cluster}")
    if size == "kitti":
        w, h = synth.KITTI_WH; L = 4; K = synth.KITTI_K; seq = kitti_seq; p4 = _p4(synth, seq, 2000)
        ctx = api.Context(K, w, h, max_frames=4, track_threads=threads, cluster_size=cluster); ctx.makeImages(0, seq.images[0]); ctx.makeImages(1, seq.images[1])
        tr = api.CoarseTracker(ctx, 0); tr.setCoarseTrackingRef(0, p4, np.zeros(len(p4), np.int32), 0.0, 1.0)
        otr = orc.CoarseTracker(w, h, L, K); otr.setCoarseTrackingRef(orc.Frame(seq.images[0], L), p4, np.zeros(len(p4), np.int32), 0.0, 1.0)
        f1 = orc.Frame(seq.images[1], L)
    else:
        from test_gpu_sizes import _seq, _tracker_pair
        S, seq = _seq(size); ctx, tr, otr, f1, L, _ = _tracker_pair(api, synth, S, seq, track_threads=threads, cluster_size=cluster)
    T0 = orc.se3_mul(orc.se3_exp([0.04, -0.02, 0.05, 0.002, -0.002, 0.001]), _tgt(synth, seq))
    rg = tr.trackNewestCoarse(1, T0, (0.0, 0.0)); assert rg["good"]
    n0 = len(otr.cloud(0)[0]); its = int(rg["iterations"][0]); m = tf.m_lm(n0, threads, cluster)
    reps = int(rg["evals"][0] // n0) - (its + 1)                              # cutoff repeats at level 0 (each doubles the cutoff)
    assert rg["evals"][0] == n0 * (its + 1 + reps) and reps >= 0
    ref = tf.Ref(otr, f1, 0, rg["T"], *rg["ab"], 20.0 * 2 ** reps, ref_b=1.0, gs=False)
    rep.check("lastRes", abs(rg["lastResiduals"][0] - ref.lastRes), ref.lastres_bound(m))
    fN = float(F(ref.n_flow)) + 0.1
    rep.check("flow[0]", abs(rg["flow"][0] - ref.rs[2]), ref.sum_bound(tf.IDX_FT, m) / fN)
    rep.check("flow[2]", abs(rg["flow"][2] - ref.rs[4]), ref.sum_bound(tf.IDX_FRT, m) / fN)
    rel = abs(rg["lastResiduals"][0] - ref.lastRes) / ref.lastRes
    rep.print(); print(f"  level 0: n = {n0}, m = {m}, lastResiduals[0] relative error {rel:.2e}")
    ctx.close()
