"""GPU (-m gpu): the device back-end on windows whose float accumulators cross the 1000-update tier (tests/ba_tiers.py) -- ba_acc_top_kernel's per-pair counters and
the shift before the TopRight / BotRight adds, ba_acc_sc_kernel's counters per accD(h,t1,t2) and per accE / accEB, its extra accHcc / accbc CTA, mode 2 of both
for marginalizePointsF.  Each window alone and installed in one batch with small windows at non-contiguous indices: the activity, HA / bA / Hsc / bsc, HS / bS,
the step, HdiF / bdSumF, optimize(6), flagPointsForRemoval and marginalizePointsF (sdv_ba_marginalize_points_batch) -> M / Mb / Msc / Mbsc and the prior HM / bM,
bit for bit against the oracle and against the reference's results stored by tests/test_ref_pin_ba_tiers.py.  The float64 bounds of tests/ba_acc_fp64.py
(normal_equations) hold on the tier windows, on the reference's live windows (tests/golden/seq_ba_ref.npz) and on the S-STRESS window of test_gpu_sizes.py; the
worst error / bound per check is printed."""
import numpy as np
import pytest
import orc
import ba_acc_fp64 as A
import ba_tiers as T
from conftest import cached_sequence
from test_ba_fp64_cpu import LAM, live_windows
from test_gpu_sequence_ba import _bit, _optimized_like_oracle
from test_ref_pin_ba_tiers import golden, golden_same, golden_value, linearized_res_to_zero
from tracker_fp64 import Report

pytestmark = pytest.mark.gpu
SYS = ("HA", "bA", "Hsc", "bsc")


@pytest.fixture(scope="module")
def world():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    seq = T.sequence()
    ctx = api.Context(synth.KITTI_K, *synth.KITTI_WH, levels=T.LEVELS, max_frames=8)
    for k in range(4):                                                      # frame handle = image index; every window shares them
        ctx.makeImages(k, seq.images[k])
    small = [synth.make_ba_window(seq, [0, 1, 2, 3], n_per_frame=50, seed=s, pose_noise=(0.005, 0.0003), match_noise=0.1, prior_scale=1e-3) for s in (21, 22)]
    yield api, ctx, small
    ctx.close()


def _solve_and_check(e, win, frames, name, rep, tag):
    """the device window e, freshly installed: linearizeAll(False) + applyRes + solveSystem(0) against the oracle, the golden (name given) and the bounds"""
    e.reset_oob(); e.linearizeAll(False); e.applyRes()
    ob = T.linearized(win, frames); rs = e.residuals()
    _bit(rs["active"], ob.residuals()["active"], f"{tag} active")
    x, HS, bS, system = e.solveSystem(0, LAM); xo, HSo, bSo = ob.solveSystem(0, LAM); so = ob.accumulate()
    got = dict(zip(SYS, system))
    for k, a, b in zip(SYS, system, so):
        _bit(a, b, f"{tag} {k}")
    _bit(HS, HSo, f"{tag} HS"); _bit(bS, bSo, f"{tag} bS"); _bit(x, xo, f"{tag} x")
    pg, po = e.points(), ob.points()
    for k in ("HdiF", "bdSumF", "step"):
        _bit(pg[k], po[k], f"{tag} {k}")
    if name is not None:
        T.check_counts(name, win, rs["active"], rs["new_state"])
        g = golden(name)
        assert golden_same(g, "active", rs["active"]), tag
        for k in SYS:
            assert golden_same(g, k, got[k]), (tag, k)
        assert golden_same(g, "HS", HS) and golden_same(g, "bS", bS), tag
        xr = golden_value(g, "x"); assert np.allclose(x, xr, rtol=1e-9, atol=1e-9 * np.abs(xr).max()), tag
        assert golden_same(g, "HdiF", pg["HdiF"]) and golden_same(g, "bdSumF", pg["bdSumF"]), tag
    A.check_equations(A.normal_equations(win, rs, pg, e.precalc, e.frames()), got, tag, rep)
    return ob


def _marg_and_check(api, es, obs, wins, sels, names, rep, tag):
    """flag_points_batch + marginalize_points_batch over the windows es (solved once, like their oracles obs): status, res_toZeroF, M / Mb / Msc / Mbsc, HM / bM"""
    sts = api.flag_points_batch(es, sels); priors0 = [e.prior() for e in es]
    api.marginalize_points_batch(es)
    for e, ob, win, sel, st, name, (HM0, bM0) in zip(es, obs, wins, sels, sts, names, priors0):
        w = f"{tag} window {e.window}"
        _bit(st, ob.flagPointsForRemoval(sel), f"{w} status")
        mo = ob.marginalizePointsF(st)
        n = e.n; M = np.zeros((n, n)); Mb = np.zeros(n); S = np.zeros((n, n)); Sb = np.zeros(n)
        e._sel(); e.ctx._ck(api.LIB.sdv_ba_get_system(e.ctx.p, M, Mb, S, Sb, np.zeros((n, n)), np.zeros(n)))
        m = dict(M=M, Mb=Mb, Msc=S, Mbsc=Sb)
        for k in m:
            _bit(m[k], mo[k], f"{w} {k}")
        r2z, lin = e.linearized(); _bit(lin, ob.res_to_zero()[1], f"{w} isLinearized"); _bit(r2z, ob.res_to_zero()[0], f"{w} res_toZeroF")
        HM1, bM1 = e.prior(); Ho, bo = ob.prior(); _bit(HM1, Ho, f"{w} HM"); _bit(bM1, bo, f"{w} bM")
        rs = e.residuals()
        dense = A.dense_marg_system(win, rs["efJ"], r2z, rs["active"], e.precalc, st)
        A.check_marginalized_points(win, m, HM0, bM0, HM1, bM1, dense, w, rep)
        if name is not None:
            T.check_marg_counts(win, rs["active"], st)
            g = golden(name)
            assert golden_same(g, "status", st) and golden_same(g, "res_to_zero", linearized_res_to_zero(r2z, lin)), w
            assert golden_same(g, "HM", HM1) and golden_same(g, "bM", bM1), w


@pytest.mark.parametrize("name", T.NAMES)
def test_tier_window_alone(world, name):
    api, ctx, _ = world; win, frames = T.window(name); rep = Report(f"device {name}")
    e = api.EnergyFunctional(ctx, win, win["kf_idx"], window=0)
    ob = _solve_and_check(e, win, frames, name, rep, name)
    if name == "schur":
        _marg_and_check(api, [e], [ob], [win], [T.marg_selection(win)], [name], rep, name)
    e = api.EnergyFunctional(ctx, win, win["kf_idx"], window=1); ob = orc.BAWindow(win, frames)
    r, ro = e.optimize(6), ob.optimize(6)
    _optimized_like_oracle(e, ob, r, ro, f"{name} optimize")
    rep.print()


def _small_selection(w):
    return ((np.asarray(w["host"]) == 0) & (np.diff(np.asarray(w["res_begin"])) >= 3)).astype(np.int32)


def test_tier_windows_batched(world):
    """all tier windows and two small ones installed by one sdv_ba_set_window_batch at non-contiguous indices, out of order"""
    api, ctx, small = world; rep = Report("device batched")
    names = list(T.NAMES) + [None, None]; wins = [T.window(n)[0] for n in T.NAMES] + small
    frames = [T.window(n)[1] for n in T.NAMES] + [T.window("schur")[1]] * 2
    W = [11, 3, 8, 14, 5, 9, 2, 12]
    es = api.EnergyFunctional.install_batch(ctx, W, wins, [w["kf_idx"] for w in wins])
    obs = [_solve_and_check(e, w, f, n, rep, f"batch {n or 'small'}") for e, w, f, n in zip(es, wins, frames, names)]
    k = [names.index("schur"), len(names) - 2, len(names) - 1]
    _marg_and_check(api, [es[i] for i in k], [obs[i] for i in k], [wins[i] for i in k], [T.marg_selection(wins[k[0]]), _small_selection(small[0]), _small_selection(small[1])],
                    ["schur", None, None], rep, "batch")
    W2 = [15, 1, 13, 6, 10, 4, 7, 0]
    es = api.EnergyFunctional.install_batch(ctx, W2, wins, [w["kf_idx"] for w in wins])
    r = api.optimize_batch(ctx, W2, 6)
    for i, (e, w, f, n) in enumerate(zip(es, wins, frames, names)):
        ob = orc.BAWindow(w, f); ro = ob.optimize(6)
        _optimized_like_oracle(e, ob, dict(rmse=r["rmse"][i], iterations=int(r["iterations"][i]), accepts=int(r["accepts"][i])), ro, f"batch {n} optimize")
    rep.print()


def test_bounds_live_windows():
    """the reference's three live windows: accumulate() within the bounds"""
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    seq = cached_sequence(200, 1000, synth.KITTI_K, synth.KITTI_WH, step=0.5)
    wins, L = live_windows(seq.wh); rep = Report("device live windows")
    ctx = api.Context(synth.KITTI_K, *seq.wh, levels=L, max_frames=24, max_kf_images=24)
    for k in sorted({k for w in wins.values() for k in w["kf_idx"]}):
        ctx.makeImages(k, seq.images[k])
    for j, (i, win) in enumerate(wins.items()):
        e = api.EnergyFunctional(ctx, win, win["kf_idx"], window=j)
        e.reset_oob(); e.linearizeAll(False); e.applyRes()
        _, _, _, system = e.solveSystem(0, LAM)
        A.check_equations(A.normal_equations(win, e.residuals(), e.points(), e.precalc, e.frames()), dict(zip(SYS, system)), f"w{i}", rep)
    ctx.close()
    rep.print()


def test_bounds_stress_window():
    """the S-STRESS window of test_gpu_sizes.py (1920x1200, 8 keyframes x 4096 points): accumulate() within the bounds"""
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    from test_gpu_sizes import SIZES
    S = SIZES["stress"]; seq = cached_sequence(S["kfs"] + 1, S["seed"], S["K"], S["wh"], beams=S["beams"]); kfs = list(range(S["kfs"]))
    win = synth.make_ba_window(seq, kfs, n_per_frame=S["n_per_frame"], seed=3, pose_noise=(0.005, 0.0003), match_noise=0.1, prior_scale=1e-3)
    ctx = api.Context(S["K"], *S["wh"], max_frames=len(kfs) + 1); rep = Report("device S-STRESS")
    for i, k in enumerate(kfs):
        ctx.makeImages(500 + i, seq.images[k])
    e = api.EnergyFunctional(ctx, win, [500 + i for i in range(len(kfs))])
    e.reset_oob(); e.linearizeAll(False); e.applyRes()
    _, _, _, system = e.solveSystem(0, LAM)
    eq = A.normal_equations(win, e.residuals(), e.points(), e.precalc, e.frames())
    A.check_equations(eq, dict(zip(SYS, system)), "stress", rep)
    print(f"\n[device S-STRESS] largest accumulator: {max(eq[1]['top'].values())} updates (top), {max(eq[1]['D'].values())} (accD)")
    ctx.close()
    rep.print()
