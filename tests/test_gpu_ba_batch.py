"""GPU (-m gpu) tests of the batched back-end install and keyframe hand-over (sdv_ba_set_window_batch, sdv_ba_set_points_batch, sdv_ba_flag_points_batch,
sdv_ba_marginalize_points_batch, sdv_ba_marginalize_frames_batch): bit-exact against a twin context driven by the single-window entries, and against the
oracle for one window whose points are permuted within their host frames; windows that never had points, installed with none; every refusal
leaves the listed windows as they were; the launches and host waits of a call do not grow with the number of windows."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence

pytestmark = pytest.mark.gpu

SIZES = {0: (1400, 360), 1: (1200, 360)}          # a KITTI-360 context (camera 0) with KITTI 00's size on camera 1
ERR_ARG, ERR_STATE = -1, -5


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _same_dict(a, b):
    return all(_same(a[k], b[k]) for k in a)


class _World:
    """two sequences (one per camera size) ingested into a context; frame id of keyframe k of camera c = 100*(c+1) + k"""

    def __init__(self, api, synth):
        self.api, self.synth = api, synth
        self.Ks = {0: tuple(synth.K360_K), 1: tuple(synth.KITTI_K)}
        self.seqs = {c: cached_sequence(8, 2100 + c, self.Ks[c], SIZES[c]) for c in (0, 1)}

    def ctx(self):
        ctx = self.api.Context(self.Ks[0], *SIZES[0], levels=4, max_frames=24, max_kf_images=24)
        ctx.setCameraSize(1, *SIZES[1])
        for c in (0, 1):
            for k in range(8):
                ctx.makeImages(self.fid(c, k), self.seqs[c].images[k], cam=c)
        return ctx

    @staticmethod
    def fid(c, k):
        return 100 * (c + 1) + k

    def window(self, c, kfs, seed, prior_scale=1e-3, kzero=False, shuffle=False, n_per_frame=120, permute=False):
        win = self.synth.make_ba_window(self.seqs[c], kfs, n_per_frame=n_per_frame, seed=seed, pose_noise=(0.005, 0.0003), match_noise=0.2, prior_scale=prior_scale)
        rng = np.random.default_rng(seed + 77)
        if permute:                                                          # a legal flattening: the points of each host frame in another order, which
            win = _permute_points(win, rng)                                  # reorders the residuals of every (host, target) pair: the sort must keep it
        if kzero:                                                            # a live CalibHessian: value_zero != value
            win["K_zero"] = np.asarray(win["K"], np.float64) * np.float64(np.float32(1) / np.float32(50)) * (1 + 1e-4 * rng.normal(size=4))
        if shuffle:                                                          # a legal flattening: residual order within each point permuted
            rb = win["res_begin"]; perm = np.arange(len(win["r_point"]))
            for p in range(len(rb) - 1):
                perm[rb[p]:rb[p + 1]] = rb[p] + rng.permutation(rb[p + 1] - rb[p])
            for k in ("r_point", "r_host", "r_target", "r_hasMatcher", "r_matcher", "r_isNew"):
                win[k] = np.ascontiguousarray(np.asarray(win[k])[perm])
        return win, [self.fid(c, k) for k in kfs]


def _permute_points(win, rng):
    host = np.asarray(win["host"]); order = np.concatenate([rng.permutation(np.nonzero(host == h)[0]) for h in range(win["nF"])]).astype(np.int64)
    out = dict(win)
    for k in ("uv", "idepth", "idepth_zero", "color", "weights", "host", "hasDepthPrior", "isFromSensor"):
        out[k] = np.ascontiguousarray(np.asarray(win[k])[order])
    rb = np.asarray(win["res_begin"]); rows = np.concatenate([np.arange(rb[p], rb[p + 1]) for p in order]).astype(np.int64)
    for k in ("r_host", "r_target", "r_hasMatcher", "r_matcher", "r_isNew"):
        out[k] = np.ascontiguousarray(np.asarray(win[k])[rows])
    cnt = np.diff(rb)[order]
    out["res_begin"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    out["r_point"] = np.repeat(np.arange(len(order)), cnt).astype(np.int32)
    return out


def _empty(win, points):
    """the window without residuals (points=True) or without points and residuals"""
    out = dict(win); nR0 = 0
    for k in ("r_point", "r_host", "r_target", "r_hasMatcher", "r_matcher", "r_isNew"):
        out[k] = np.asarray(win[k])[:nR0]
    if not points:
        for k in ("uv", "idepth", "idepth_zero", "color", "weights", "host", "hasDepthPrior", "isFromSensor"):
            out[k] = np.asarray(win[k])[:0]
    out["res_begin"] = np.zeros(len(out["uv"]) + 1, np.int32)
    return out


# (camera, keyframes, prior scale, value_zero != value, shuffled residuals)
MIXED = [(1, [0, 1, 2, 3, 4, 5, 6], 1e-3, False, False), (0, [1, 2, 4, 5, 7], 1e-3, True, True), (1, [2, 5], 0.0, False, False),
         (0, [0, 1, 2, 3, 4, 5, 6, 7], 1e-2, False, True), (1, [0, 2, 4, 6], 1e-3, True, False), (0, [3, 4, 5], 0.0, False, False),
         (1, [1, 3, 5, 6, 7], 1e-3, False, True), (0, [0, 1, 2, 3, 4, 5], 1e-3, True, False)]
WINDOWS = [5, 0, 9, 2, 7, 1, 3, 12]                    # any indices, in any order


def _install(api, ctx, twin, W, wins, ids):
    eb = api.EnergyFunctional.install_batch(ctx, W, wins, ids)
    es = [api.EnergyFunctional(twin, w, i, window=k) for k, w, i in zip(W, wins, ids)]
    return eb, es


def _compare_windows(eb, es):
    for a, b in zip(eb, es):
        assert (a.nF, a.nP, a.nR, a.n) == (b.nF, b.nP, b.nR, b.n)
        assert _same_dict(a.frames(), b.frames()), a.window
        if a.nP:
            assert _same_dict(a.points(), b.points()) and _same_dict(a.residuals(), b.residuals()), a.window
        for h, t in ((0, a.nF - 1), (a.nF - 1, 0)):
            if h != t:
                pa, pb = a.precalc(h, t), b.precalc(h, t)
                assert all(_same(pa[k], pb[k]) for k in pa), (a.window, h, t)
        assert all(_same(x, y) for x, y in zip(a.prior(), b.prior())), a.window


def test_mixed_install_bit_exact():
    api, synth = _mods(); world = _World(api, synth)
    ctx, twin = world.ctx(), world.ctx()
    specs = [world.window(c, kfs, 40 + i, ps, kz, sh) for i, (c, kfs, ps, kz, sh) in enumerate(MIXED)]
    wins, ids = [s[0] for s in specs], [s[1] for s in specs]
    eb, es = _install(api, ctx, twin, WINDOWS, wins, ids)
    _compare_windows(eb, es)
    for a, b in zip(eb, es):                                                 # one solveSystem step per window
        a.linearizeAll(False); b.linearizeAll(False); a.applyRes(); b.applyRes()
        xa, Ha, ba, sa = a.solveSystem(0, 0.0); xb, Hb, bb, sb = b.solveSystem(0, 0.0)
        assert _same(xa, xb) and _same(Ha, Hb) and _same(ba, bb) and all(_same(u, v) for u, v in zip(sa, sb)), a.window
    eb, es = _install(api, ctx, twin, WINDOWS, wins, ids)                    # re-install over the used windows, then the Gauss-Newton loop
    ra, rb = api.optimize_batch(ctx, WINDOWS, 6), api.optimize_batch(twin, WINDOWS, 6)
    assert all(_same(ra[k], rb[k]) for k in ("rmse", "iterations", "accepts")) and (ra["accepts"] > 0).all()
    _compare_windows(eb, es)
    ctx.close(); twin.close()


def _select(win, marg_host, every):
    sel = (win["host"] == marg_host).astype(np.int32); sel[::every] = 1
    sel[win["host"] == win["nF"] - 1] = 0
    return sel


def test_two_keyframe_steps_against_single_calls_and_oracle():
    api, synth = _mods(); world = _World(api, synth)
    ctx, twin = world.ctx(), world.ctx()
    # (camera, keyframes, frames eliminated in order in each step: 0, 1 or 2 per window, the second one at a shifted index)
    plan = [(1, [0, 1, 2, 3, 4, 5, 6], [2, 0]), (0, [1, 2, 4, 5, 7], [1]), (1, [2, 3, 5], []), (0, [0, 1, 2, 3, 4, 5, 6, 7], [3, 3]),
            (1, [0, 2, 4, 6], [0]), (0, [3, 4, 5, 6], []), (1, [1, 3, 5, 6, 7], [2, 1]), (0, [0, 1, 2, 3, 4, 5], [1]), (1, [4, 5], [])]
    W = list(range(len(plan)))[::-1]
    # window 0, which the oracle checks as well, has its points permuted within each host and its residuals shuffled within each point
    specs = [world.window(c, kfs, 60 + i, 1e-3, i % 3 == 1, i % 2 == 1 or i == 0, permute=(i == 0)) for i, (c, kfs, _) in enumerate(plan)]
    wins, ids = [s[0] for s in specs], [s[1] for s in specs]
    for step in range(2):
        eb, es = _install(api, ctx, twin, W, wins, ids)
        ra, rb = api.optimize_batch(ctx, W, 6), api.optimize_batch(twin, W, 6)
        assert all(_same(ra[k], rb[k]) for k in ("rmse", "iterations", "accepts"))
        if step == 0:                                                        # window 0 against the oracle: its loop, flags and priors
            L = api.pyr_levels(*SIZES[plan[0][0]])
            ob = orc.BAWindow(wins[0], [orc.Frame(world.seqs[plan[0][0]].images[k], L) for k in plan[0][1]])
            ro = ob.optimize(6)
            assert (ro["iterations"], ro["accepts"]) == (ra["iterations"][0], ra["accepts"][0])
        _compare_windows(eb, es)
        sels = [_select(w, min(1, w["nF"] - 2), 3 + i % 3) for i, w in enumerate(wins)]
        sa = api.flag_points_batch(eb, sels); sb = [e.flagPointsForRemoval(s) for e, s in zip(es, sels)]
        assert all(_same(x, y) for x, y in zip(sa, sb))
        if step == 0:
            so = ob.flagPointsForRemoval(sels[0]); assert _same(so, sa[0])
        api.marginalize_points_batch(eb); mb = [e.marginalizePointsF() for e in es]
        for a, m in zip(eb, mb):
            HA = np.zeros((a.n, a.n)); bA = np.zeros(a.n); Hs = np.zeros((a.n, a.n)); bs = np.zeros(a.n); d1 = np.zeros((a.n, a.n)); d2 = np.zeros(a.n)
            a._sel(); a.ctx._ck(api.LIB.sdv_ba_get_system(a.ctx.p, HA, bA, Hs, bs, d1, d2))
            assert _same(HA, m["M"]) and _same(bA, m["Mb"]) and _same(Hs, m["Msc"]) and _same(bs, m["Mbsc"]), a.window
        _compare_windows(eb, es)
        elim = [p[2] for p in plan]
        pa = api.marginalize_frames_batch(eb, elim)
        for e, el in zip(es, elim):
            for x in el:
                e.marginalizeFrame(x)
        for a, b, (H, bM) in zip(eb, es, pa):
            Hb, bb = b.prior(); assert _same(H, Hb) and _same(bM, bb) and (a.nF, a.n, a.nP, a.nR) == (b.nF, b.n, b.nP, b.nR)
            assert all(_same(x, y) for x, y in zip(a.prior(), (Hb, bb)))
        if step == 0:
            ob.marginalizePointsF(so)
            for x in elim[0]:
                ob.marginalizeFrame(x)
            assert all(_same(x, y) for x, y in zip(ob.prior(), pa[0]))
        # the next keyframe step: each window re-flattened without its eliminated frames, carrying its prior
        nxt = []
        for i, ((c, kfs, el), (H, bM)) in enumerate(zip(plan, pa)):
            kk = list(kfs)
            for x in el:
                kk.pop(x)
            w, f = world.window(c, kk, 90 + i, 0.0, i % 3 == 1, i % 2 == 1); w["HM"] = H; w["bM"] = bM
            nxt.append((w, f))
        plan = [(c, list(w["kf_idx"]), el) for (c, _, el), (w, _) in zip(plan, nxt)]
        wins, ids = [s[0] for s in nxt], [s[1] for s in nxt]
    eb, es = _install(api, ctx, twin, W, wins, ids)
    ra, rb = api.optimize_batch(ctx, W, 6), api.optimize_batch(twin, W, 6)
    assert all(_same(ra[k], rb[k]) for k in ("rmse", "iterations", "accepts"))
    _compare_windows(eb, es)
    ctx.close(); twin.close()


def _state(efs):
    out = []
    for e in efs:
        s = dict(frames=e.frames(), prior=e.prior(), n=(e.nF, e.nP, e.nR))
        if e.nP:
            s.update(points=e.points(), residuals=e.residuals())
        out.append(s)
    return out


def _same_state(a, b):
    for x, y in zip(a, b):
        assert x["n"] == y["n"] and _same_dict(x["frames"], y["frames"]) and all(_same(u, v) for u, v in zip(x["prior"], y["prior"]))
        if "points" in x:
            assert _same_dict(x["points"], y["points"]) and _same_dict(x["residuals"], y["residuals"])
    return True


def _set_points(api, ctx, W, k):
    return api.LIB.sdv_ba_set_points_batch(ctx.p, len(W), np.ascontiguousarray(W, np.int32), k["p_begin"], k["r_begin"], k["uv"], k["idepth"], k["idepth_zero"],
                                           k["color"], k["weights"], k["host"], k["hasDepthPrior"], k["isFromSensor"], k["res_begin"], k["r_point"], k["r_host"],
                                           k["r_target"], k["r_hasMatcher"], k["r_matcher"], k["r_isNew"])


def _set_window(api, ctx, W, k, frame_ids=None):
    ptr = lambda a: None if a is None else a.ctypes.data
    return api.LIB.sdv_ba_set_window_batch(ctx.p, len(W), np.ascontiguousarray(W, np.int32), k["f_begin"],
                                           np.ascontiguousarray(k["frame_ids"] if frame_ids is None else frame_ids, np.uint64), k["T_eval"], k["state"],
                                           k["state_zero"], k["ab_exposure"], k["frameID"], k["frameEnergyTH"], k["K"], ptr(k["K_zero"]), ptr(k["HM"]), ptr(k["bM"]))


def test_refusals_leave_every_window_unchanged():
    api, synth = _mods(); world = _World(api, synth)
    ctx = world.ctx()
    specs = [world.window(1, [0, 1, 2, 3], 11), world.window(0, [2, 3, 4], 12), world.window(1, [5, 6], 13, n_per_frame=60)]
    wins, ids = [s[0] for s in specs], [s[1] for s in specs]
    W = [4, 1, 6]
    eb = api.EnergyFunctional.install_batch(ctx, W, wins, ids)
    before = _state(eb)
    big, _ = world.window(1, [5, 6], 14, n_per_frame=600)                   # window 6 would need a larger pool
    for what in ("host", "residual", "duplicate", "span", "monotone", "grow"):
        ws = [dict(w) for w in wins]; i = 1
        if what == "host":
            h = ws[1]["host"].copy(); p = int(np.nonzero(h > 0)[0][0]); h[p], h[p - 1] = h[p - 1], h[p]; ws[1]["host"] = h
        elif what == "residual":
            t = ws[1]["r_host"].copy(); t[len(t) // 2] = (t[len(t) // 2] + 1) % ws[1]["nF"]; ws[1]["r_host"] = t
        elif what == "duplicate":
            rb = ws[1]["res_begin"]; p = int(np.nonzero(np.diff(rb) >= 2)[0][0]); t = ws[1]["r_target"].copy(); t[rb[p] + 1] = t[rb[p]]; ws[1]["r_target"] = t
        elif what == "span":
            rb = ws[1]["res_begin"].copy(); rb[-1] -= 1; ws[1]["res_begin"] = rb
        elif what == "monotone":
            rb = ws[1]["res_begin"].copy(); p = len(rb) // 2; rb[p] = rb[p + 1] + 1; ws[1]["res_begin"] = rb
        else:
            ws[2] = big; t = ws[1]["r_host"].copy(); t[0] = (t[0] + 1) % ws[1]["nF"]; ws[1]["r_host"] = t
        k = api.pack_ba_windows(ws, ids)
        assert _set_points(api, ctx, W, k) == ERR_ARG, what
        msg = api.LIB.sdv_last_error(ctx.p).decode(); assert f"window {W[i]}" in msg, (what, msg)
        assert _same_state(before, _state(eb)), what
    k = api.pack_ba_windows(wins, ids)
    assert _set_points(api, ctx, [4, 1, 4], api.pack_ba_windows([wins[0], wins[1], wins[0]], [ids[0], ids[1], ids[0]])) == ERR_ARG   # listed twice
    assert _set_window(api, ctx, [4, 1, 4], api.pack_ba_windows([wins[0], wins[1], wins[0]], [ids[0], ids[1], ids[0]])) == ERR_ARG
    ctx.makeImages(999, world.seqs[1].images[7], cam=1)                   # a frame only a refused call names
    f = k["frame_ids"].copy(); f[-1] = 4242                                  # an unknown frame in the last window
    assert _set_window(api, ctx, W, k, f) != 0
    f = k["frame_ids"].copy(); f[-1] = 999; f[0] = world.fid(0, 0)          # mixed sizes in window 4, the new frame in window 6
    assert _set_window(api, ctx, W, k, f) == ERR_ARG
    assert _same_state(before, _state(eb))
    for fid in [x for s in ids for x in s]:                                  # the windows' frames are still pinned, the refused call's new frame is not
        assert api.LIB.sdv_frame_release(ctx.p, fid) == ERR_STATE
    assert api.LIB.sdv_frame_release(ctx.p, 999) == 0
    WW = np.ascontiguousarray(W, np.int32); H = np.zeros(10000); b = np.zeros(200)
    for kb, idx in (([0, 1, 1, 2], [0, 4]), ([0, 0, 0, 2], [0, 0]), ([0, 1, 2, 3], [0, 2, -1])):   # out of range; down to zero frames; negative
        rc = api.LIB.sdv_ba_marginalize_frames_batch(ctx.p, 3, WW, np.array(kb, np.int32), np.array(idx, np.int32), H.ctypes.data, b.ctypes.data)
        assert rc == ERR_ARG, (kb, idx)
    assert _same_state(before, _state(eb))
    for fid in [x for s in ids for x in s]:
        assert api.LIB.sdv_frame_release(ctx.p, fid) == ERR_STATE
    ctx.close()


def test_fresh_windows_without_points_or_residuals_in_a_batch():
    """windows that never had points, installed in one batch with zero points or zero residuals, next to a full one: the same state as the single
    entries leave in a twin context, and both contexts stay usable"""
    api, synth = _mods(); world = _World(api, synth)
    ctx, twin = world.ctx(), world.ctx()
    (w0, i0), (w1, i1), (w2, i2) = world.window(1, [0, 1, 2, 3], 21), world.window(0, [1, 2, 3], 22), world.window(1, [4, 5, 6], 23)
    wins, ids, W = [w0, _empty(w1, False), _empty(w2, True)], [i0, i1, i2], [3, 8, 4]
    eb, es = _install(api, ctx, twin, W, wins, ids)
    assert [e.nP for e in eb] == [len(w0["uv"]), 0, len(w2["uv"])] and [e.nR for e in eb] == [len(w0["r_point"]), 0, 0]
    _compare_windows(eb, es)
    ra, rb = api.optimize_batch(ctx, [3], 6), api.optimize_batch(twin, [3], 6)
    assert all(_same(ra[k], rb[k]) for k in ("rmse", "iterations", "accepts")) and ra["accepts"][0] > 0
    assert api.LIB.sdv_ba_flag_points_batch(ctx.p, 2, np.array([3, 8], np.int32), np.zeros(len(w0["uv"]), np.int32), None) == ERR_STATE
    pa = api.marginalize_frames_batch(eb, [[1], [0], []])
    for e, x in zip(es, [[1], [0], []]):
        for k in x:
            e.marginalizeFrame(k)
    assert all(_same(H, b.prior()[0]) and _same(bM, b.prior()[1]) for (H, bM), b in zip(pa, es))
    eb, es = _install(api, ctx, twin, W, [w0, w1, w2], ids)                   # the same windows with their points: pools grow from the empty ones
    _compare_windows(eb, es)
    ctx.close(); twin.close()


def test_launches_and_host_waits_do_not_grow_with_windows():
    api, synth = _mods(); world = _World(api, synth)
    ctx = world.ctx()
    specs = [world.window(i % 2, [0, 1, 2, 3, 4], 30 + i, n_per_frame=60) for i in range(8)]
    counts = []
    for n in (8, 2, 8):                                                      # the first pass builds the frames' level-0 texels and grows the staging
        wins, ids = [s[0] for s in specs[:n]], [s[1] for s in specs[:n]]; row = []

        def cost(f):
            l0, w0 = ctx.launch_count(), ctx.ba_host_wait_count(); r = f(); row.append((ctx.launch_count() - l0, ctx.ba_host_wait_count() - w0)); return r
        eb = cost(lambda: api.EnergyFunctional.install_batch(ctx, list(range(n)), wins, ids))
        cost(lambda: api.flag_points_batch(eb, [_select(w, 1, 3) for w in wins]))
        cost(lambda: api.marginalize_points_batch(eb))
        cost(lambda: api.marginalize_frames_batch(eb, [[1, 0]] * n))
        counts.append(row)
    assert counts[1] == counts[2], counts
    assert [w for _, w in counts[1]] == [3, 1, 1, 1], counts                 # set_window 1 + set_points 2, then one wait per hand-over call
    ctx.close()
