"""GPU tests (-m gpu) of cameras of different pyramid depths in one context (sdv_set_camera_levels, sdv_tracker_track_batch_levels).

One 1400x1024 context stores every frame at 5 levels.  Its cameras, each at its own pyrLevelsUsed:
  camera 0  1400x1024, set to 4 levels
  camera 1  KITTI-CARLA 1392x1024 (calib/kitti_carla.txt), 5 levels
  camera 2  KITTI-360 1400x360, 4 levels
  camera 3  KITTI 00 1200x360, 4 levels
  camera 4  1244x356, 3 levels (its pyr_levels: level 2 is 311x89)
The per-camera reference is a fresh context created at that camera's own (w, h, levels): every job of a mixed batch must equal it bit for bit, and the oracle
run at that depth within the tolerances of the single-context tests."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from test_undistort import CALIBS, _check_levels

pytestmark = pytest.mark.gpu

CTX_WH, CTX_L = (1400, 1024), 5
SIZES = [(1400, 1024), (1392, 1024), (1400, 360), (1200, 360), (1244, 356)]
LEVELS = [4, 5, 4, 4, 3]
N = 6                                                      # frames per camera
KFS = [0, 1, 2, 3]                                         # map keyframes; frame 3 is the tracking reference
ERR_ARG, ERR_STATE = -1, -5


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _Ks(synth):
    carla = tuple(float(v) for v in CALIBS["carla"].split()[1:5])
    return [(900.0, 900.0, 699.5, 511.5), carla, tuple(synth.K360_K), tuple(synth.KITTI_K), (702.5, 698.0, 611.0, 171.5)]


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _mixed(api, synth, **kw):
    """the 5-level context with every camera at its size and depth; camera 0 keeps the context calibration"""
    ctx = api.Context(_Ks(synth)[0], *CTX_WH, levels=CTX_L, **kw)
    for c in range(1, 5):
        ctx.setCameraSize(c, *SIZES[c])
    for c in range(5):
        ctx.setCameraLevels(c, LEVELS[c])
    return ctx


def filtered_order(order, c):
    """the context grid's cell_order as camera c's job walks it (sdv_b200.h, sdv_reproject_map_batch)"""
    ncols = -(-CTX_WH[0] // 25); jc, jr = -(-SIZES[c][0] // 25), -(-SIZES[c][1] // 25)
    return np.array([(k // ncols) * jc + k % ncols for k in order if k % ncols < jc and k // ncols < jr], np.int32)


class Cam:
    """one camera: its rendered sequence, map, reference cloud, oracle frames at its depth"""

    def __init__(self, synth, c, K):
        self.c, self.K, self.wh, self.L = c, K, SIZES[c], LEVELS[c]
        self.seq = seq = cached_sequence(N, 8101 + 97 * c, K, self.wh)
        self.ids = [1000 * (c + 1) + i for i in range(N)]
        self.pts, self.hT, self.hab = synth.make_map(seq, KFS, n_per_frame=400, seed=3)
        self.poses = np.array([np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(N)])
        ref = synth.select_points(seq.images[3], seq.clouds[3], 2000)
        self.p4 = np.concatenate([ref, np.full((len(ref), 1), 1e-3, np.float32)], 1).astype(np.float32); self.rh = np.zeros(len(self.p4), np.int32)
        self.Tgt = orc.se3_from_rt(*synth.rel_pose(seq.R[3], seq.t[3], seq.R[4], seq.t[4]))
        self.of = [orc.Frame(im, self.L) for im in seq.images]

    def load(self, api, ctx, slots, cam):
        ims = [np.ascontiguousarray(im, np.float32) for im in self.seq.images]
        ctx.makeImagesBatch(self.ids, [a.ctypes.data for a in ims], cams=[cam] * N); ctx.sync()
        rp = api.Reprojector(ctx)
        for s in slots:
            api.CoarseTracker(ctx, s).setCoarseTrackingRef(self.ids[3], self.p4, self.rh)
            rp.setMap(s, [self.ids[k] for k in KFS], self.hT, self.hab, self.pts)
        return rp

    def fresh(self, api, **kw):
        f = api.Context(self.K, *self.wh, levels=self.L, n_tracker_slots=2, max_frames=N + 2, max_kf_images=N + 2, **kw)
        return f, self.load(api, f, [0, 1], 0)


def _contexts(api, synth, cams, **kw):
    """the mixed context (slots 2c, 2c+1 -> camera c) and one fresh context per camera (slots 0, 1)"""
    mixed = _mixed(api, synth, n_tracker_slots=10, max_frames=5 * N + 2, max_kf_images=12, **kw)
    mixed.setCalibSlots(list(range(2, 10)), [cams[s // 2].K for s in range(2, 10)], cams=[s // 2 for s in range(2, 10)])
    mrp = [cam.load(api, mixed, [2 * c, 2 * c + 1], c) for c, cam in enumerate(cams)][0]
    return mixed, mrp, [cam.fresh(api, **kw) for cam in cams]


@pytest.fixture(scope="module")
def setup():
    api, synth = _mods()
    cams = [Cam(synth, c, K) for c, K in enumerate(_Ks(synth))]
    mixed, mrp, fresh = _contexts(api, synth, cams)
    yield api, synth, cams, mixed, mrp, fresh
    mixed.close()
    for f, _ in fresh:
        f.close()


# ------------------------------------------------------------------------------------------------ ingest
def test_ingest_levels_below_each_depth(setup):
    """levels below a camera's depth equal a context of its own depth and the oracle's makeImages; deeper levels are refused"""
    api, synth, cams, mixed, mrp, fresh = setup
    for c, cam in enumerate(cams):
        f = fresh[c][0]
        for k in (0, 4):
            _check_levels(api, mixed, cam.ids[k], cam.seq.images[k].astype(np.float32), cam.L)
            for l in range(cam.L):
                a, b = mixed.frameLevel(cam.ids[k], l), f.frameLevel(cam.ids[k], l)
                assert _same(a[0], b[0]) and _same(a[1], b[1]), (c, k, l)
        for l in range(cam.L, CTX_L + 1):
            assert api.LIB.sdv_frame_download(mixed.p, cam.ids[0], l, None, None) == ERR_ARG, (c, l)
            with pytest.raises(api.SdvError):
                mixed.frameLevel(cam.ids[0], l)


# ------------------------------------------------------------------------------------------------ tracker
def _track_inits(cam, k):
    xis = ([0, 0, 0, 0, 0, 0], [0.01, -0.005, 0.02, 1e-3, -1e-3, 5e-4])
    return np.stack([orc.se3_mul(orc.se3_exp(xi), cam.Tgt) for xi in xis[:k]])


def test_reference_clouds_and_calcres_every_level(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    for c, cam in enumerate(cams):
        otr = orc.CoarseTracker(*cam.wh, cam.L, cam.K); otr.setCoarseTrackingRef(cam.of[3], cam.p4, cam.rh)
        T = _track_inits(cam, 2)[1]
        for j in (0, 1):
            tm, tf = api.CoarseTracker(mixed, 2 * c + j), api.CoarseTracker(fresh[c][0], j)
            assert tm.levels == cam.L
            for l in range(cam.L):
                a, b, o = tm.cloud(l), tf.cloud(l), otr.cloud(l)
                assert len(a[0]) > 0 and all(_same(x, y) for x, y in zip(a, b)) and all(_same(x, y) for x, y in zip(a, o)), (c, j, l)
                rm = tm.calcRes(cam.ids[4], l, T, 0.02, -1.0, 20.0); Hm, bm = tm.calcGSSSE(l)
                rf = tf.calcRes(cam.ids[4], l, T, 0.02, -1.0, 20.0); Hf, bf = tf.calcGSSSE(l)
                assert _same(rm, rf) and _same(Hm, Hf) and _same(bm, bf), (c, j, l)
                ro = otr.calcRes(cam.of[4], l, T, 0.02, -1.0, 20.0); Ho, bo = otr.calcGSSSE(l, T, 0.02, -1.0)
                assert rm[1] == ro[1] and np.isclose(rm[0], ro[0], rtol=2e-5) and np.allclose(rm[2:5], ro[2:5], rtol=1e-4, atol=1e-7), (c, l)
                assert np.linalg.norm(Hm - Ho) <= 2e-5 * np.linalg.norm(Ho) and np.linalg.norm(bm - bo) <= 2e-5 * np.linalg.norm(bo) + 1e-9, (c, l)
            for l in range(cam.L, CTX_L):
                for call in (lambda: api.LIB.sdv_tracker_get_cloud(mixed.p, 2 * c + j, l, api.C.byref(api.C.c_int(0)), None, None, None, None),
                             lambda: api.LIB.sdv_tracker_calc_res(mixed.p, 2 * c + j, cam.ids[4], l, np.ascontiguousarray(T), 0.0, 0.0, 20.0, np.zeros(6))):
                    assert call() == ERR_ARG, (c, j, l)


def _track_all(api, cams, mixed, fresh, oracle=False):
    """every slot of the mixed context in ONE launch, each job at its own depth, vs each camera's slots in its fresh context"""
    T = np.concatenate([_track_inits(cam, 2) for cam in cams]); ab = np.zeros((10, 2)); ab[1::2] = [0.02, 1.0]
    T0, ab0 = T.copy(), ab.copy()
    rm = mixed.trackBatch(list(range(10)), [cams[s // 2].ids[4] for s in range(10)], T, ab)
    for c, cam in enumerate(cams):
        sl = slice(2 * c, 2 * c + 2); Tf, abf = T0[sl].copy(), ab0[sl].copy()
        rf = fresh[c][0].trackBatch([0, 1], [cam.ids[4]] * 2, Tf, abf)
        assert np.array_equal(T[sl], Tf) and np.array_equal(ab[sl], abf), c
        for key in ("good", "flow", "iterations", "accepts", "evals"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        assert _same(rm["lastResiduals"][sl], rf["lastResiduals"]), c
        assert rf["good"].all() and (rm["iterations"][sl, cam.L - 1] > 0).all() and not rm["iterations"][sl, cam.L:].any() and not rm["evals"][sl, cam.L:].any(), c
        if oracle:
            otr = orc.CoarseTracker(*cam.wh, cam.L, cam.K); otr.setCoarseTrackingRef(cam.of[3], cam.p4, cam.rh)
            for j in (0, 1):
                ro = otr.trackNewestCoarse(cam.of[4], T0[2 * c + j], ab0[2 * c + j], cam.L - 1)
                assert ro["good"] and np.array_equal(rm["iterations"][2 * c + j], ro["iterations"]) and np.array_equal(rm["accepts"][2 * c + j], ro["accepts"]), (c, j)
                assert np.abs(orc.se3_log(orc.se3_mul(T[2 * c + j], orc.se3_inv(ro["T"])))).max() < 1e-5 and np.allclose(ab[2 * c + j], ro["ab"], atol=1e-3), (c, j)
    return T, ab, rm


def test_track_batch_mixed_depths(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    T, ab, rm = _track_all(api, cams, mixed, fresh, oracle=True)
    # a per-job sequence naming each job's depth - 1 is the default; a scalar below every depth starts every job there
    n = 10; ids = [cams[s // 2].ids[4] for s in range(n)]; T0 = np.concatenate([_track_inits(cam, 2) for cam in cams]); ab0 = np.zeros((n, 2)); ab0[1::2] = [0.02, 1.0]
    Ta, aba = T0.copy(), ab0.copy(); ra = mixed.trackBatch(list(range(n)), ids, Ta, aba, coarsest=[LEVELS[s // 2] - 1 for s in range(n)])
    assert _same(Ta, T) and _same(aba, ab) and all(_same(ra[k], rm[k]) for k in rm)
    rb = mixed.trackBatch(list(range(n)), ids, T0.copy(), ab0.copy(), coarsest=2)
    assert not rb["iterations"][:, 3:].any() and (rb["iterations"][:, 2] > 0).all()


@pytest.mark.parametrize("kw", [dict(track_threads=64), dict(cluster_size=8, track_threads=256)], ids=["threads64", "cluster8"])
def test_track_batch_mixed_depths_launch_configs(setup, kw):
    api, synth, cams = setup[:3]
    mixed, mrp, fresh = _contexts(api, synth, cams, **kw)
    _track_all(api, cams, mixed, fresh)
    mixed.close()
    for f, _ in fresh:
        f.close()


def test_track_new_coarse_batch_mixed_depths(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    order = np.random.default_rng(4).permutation(mrp.n_cells).astype(np.int32)

    def jobs_of(cam, slots):
        P = cam.poses; base = dict(frame=cam.ids[5], sprelast_c2w=P[3], slast_c2w=P[4], lastF_c2w=P[3], aff_last=[0.0, 0.0], poses_valid=1)
        return [dict(base, slot=slots[0], lastCoarseRMSE=[100.0] * 5),                           # healthy: one try
                dict(base, slot=slots[1], lastCoarseRMSE=[1e-3] * 5)]                            # all 31 hypotheses
    jm = sum([jobs_of(cam, [2 * c, 2 * c + 1]) for c, cam in enumerate(cams)], [])
    rm = api.trackNewCoarseBatch(mixed, jm, cell_order=order)
    for c, cam in enumerate(cams):
        fo = filtered_order(order, c)
        rf = api.trackNewCoarseBatch(fresh[c][0], jobs_of(cam, [0, 1]), cell_order=fo)
        for k, g in enumerate(rf):
            for key in g:
                assert _same(rm[2 * c + k][key], g[key]), (c, k, key)
        assert [r["tries"] for r in rf] == [1, 31] and all(r["n_matches"] > 10 for r in rf), c
        otr = orc.CoarseTracker(*cam.wh, cam.L, cam.K); otr.setCoarseTrackingRef(cam.of[3], cam.p4, cam.rh)
        for k, j in enumerate(jobs_of(cam, [0, 1])):
            o = orc.track_new_coarse(otr, cam.of[5], cam.K, [cam.of[i] for i in KFS], cam.hT, cam.hab, cam.pts, j["sprelast_c2w"], j["slast_c2w"], j["lastF_c2w"],
                                     j["aff_last"], j["poses_valid"], j["lastCoarseRMSE"], cell_order=fo)
            g = rf[k]
            assert g["tries"] == o["tries"] and g["have_one_good"] == o["have_one_good"] and g["n_matches"] == o["n_matches"], (c, k)
            assert np.allclose(g["lastCoarseRMSE"], o["lastCoarseRMSE"], rtol=1e-4, equal_nan=True) and np.abs(g["camToWorld"] - o["camToWorld"]).max() < 1e-6, (c, k)


# ------------------------------------------------------------------------------------------------ Reprojector search-level cap
def zoom_map(api, cam, n=900, seed=5):
    """map points on the keyframes at 10 m, seen by a target camera 8.6 m further along the optical axis: every patch is magnified ~7x, so
    getBestSearchLevel's determinant is ~50 > 3*4^2 and wants level 3, past the 3-level camera's cap"""
    rng = np.random.default_rng(seed); w, h = cam.wh; K = cam.K; pts = np.zeros(n, api.MAP_PT_DTYPE)
    pts["u"] = np.round(K[2] + rng.uniform(-0.06, 0.06, n) * w); pts["v"] = np.round(K[3] + rng.uniform(-0.06, 0.06, n) * h)
    pts["idepth"] = 0.1; pts["host"] = np.sort(rng.integers(0, len(KFS), n)); pts["type"] = (rng.uniform(size=n) < 0.3).astype(np.int32)
    hT = np.tile(np.array([1.0, 0, 0, 0, 0, 0, 0]), (len(KFS), 1)); cur = np.array([1.0, 0, 0, 0, 0, 0, 8.6])
    return pts, hT, cur


def test_reproject_and_refine_cap_at_camera_depth(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    cam = cams[4]; pts, hT, cur = zoom_map(api, cam); hab = np.zeros((len(KFS), 2)); hid = [cam.ids[k] for k in KFS]
    deep = api.Context(cam.K, *cam.wh, levels=CTX_L, n_tracker_slots=2, max_frames=N + 2, max_kf_images=N + 2)
    ims = [np.ascontiguousarray(im, np.float32) for im in cam.seq.images]; deep.makeImagesBatch(cam.ids, [a.ctypes.data for a in ims]); deep.sync()
    drp = api.Reprojector(deep); frp = fresh[4][1]
    order = np.random.default_rng(2).permutation(mrp.n_cells).astype(np.int32); fo = filtered_order(order, 4)
    for rp, s in ((mrp, 8), (frp, 0), (drp, 0)):
        rp.setMap(s, hid, hT, hab, pts)
    for tgt in (4, 5):
        Tc = cur.copy(); args = lambda s: ([s, 2], [cam.ids[tgt], cams[1].ids[tgt]], np.stack([Tc, cams[1].poses[tgt]]))
        gm = mrp.reprojectMapBatch(*args(8), cell_order=order, max_matches=400)
        gf = frp.reprojectMap(0, cam.ids[tgt], Tc, cell_order=fo, max_matches=400)
        gd = drp.reprojectMap(0, cam.ids[tgt], Tc, cell_order=fo, max_matches=400)
        o = orc.reproject_map(*cam.wh, cam.L, cam.K, [cam.of[k] for k in KFS], hT, hab, cam.of[tgt], Tc, [0.0, 0.0], pts, cell_order=fo, max_matches=400)
        of5 = [orc.Frame(im, CTX_L) for im in cam.seq.images]                                 # the oracle at 5 levels needs frames of 5 levels
        od = orc.reproject_map(*cam.wh, CTX_L, cam.K, [of5[k] for k in KFS], hT, hab, of5[tgt], Tc, [0.0, 0.0], pts, cell_order=fo, max_matches=400)
        assert _same(gm[0][0], gf[0]) and _same(gm[0][1], gf[1]) and _same(gf[0], o[0]) and _same(gf[1], o[1]), tgt
        assert _same(gd[0], od[0]) and _same(gd[1], od[1]), tgt
        assert len(o[0]) > 5 and not (_same(gd[0], gf[0]) and _same(gd[1], gf[1])), (tgt, len(o[0]), len(od[0]))   # the cap is reached
        fk = [cams[1].ids[k] for k in KFS]                                                    # the 5-level job of the same batch equals its own context
        g1 = fresh[1][1]; g1.setMap(1, fk, cams[1].hT, cams[1].hab, cams[1].pts)
        r1 = g1.reprojectMap(1, cams[1].ids[tgt], cams[1].poses[tgt], cell_order=filtered_order(order, 1), max_matches=400)
        assert _same(gm[1][0], r1[0]) and _same(gm[1][1], r1[1]) and len(r1[0]) > 10
        fm = mrp.refineBatch([8, 2], [cam.ids[tgt], cams[1].ids[tgt]], np.stack([Tc, cams[1].poses[tgt]]), cell_order=order, max_matches=150)
        ff = frp.refineBatch([0], [cam.ids[tgt]], Tc[None], cell_order=fo, max_matches=150)
        fd = drp.refineBatch([0], [cam.ids[tgt]], Tc[None], cell_order=fo, max_matches=150)
        for key in ("T", "n_matches", "res", "iterations", "accepts"):
            assert np.array_equal(fm[key][:1], ff[key]), (tgt, key)
        assert not all(np.array_equal(ff[k], fd[k]) for k in ("T", "n_matches")), tgt
    for rp, s in ((mrp, 8), (frp, 0)):                                                         # the fixture's maps
        rp.setMap(s, hid, cam.hT, cam.hab, cam.pts)
    deep.close()


# ------------------------------------------------------------------------------------------------ keyframe rate
def test_keyframe_step_on_every_camera_with_three_levels(setup):
    """makeNewTraces + activation of one keyframe per camera (every depth >= 3), in one batch: each equals a context of the camera's own size and depth"""
    api, synth, cams, mixed, mrp, fresh = setup
    cs = [4, 1, 0, 3, 2]; n = len(cs)
    ps = api.PixelSelector(mixed, n, api.random_pattern(*CTX_WH), cams=cs)
    clouds = [cams[c].seq.clouds[0] for c in cs]; dens = [900.0 + 100 * j for j in range(n)]
    res, num = ps.makeNewTracesBatch(list(range(n)), [cams[c].ids[0] for c in cs], clouds, [0.5 * d for d in dens], dens, [1] * n, cap=1 << 16)
    rng = np.random.default_rng(1); seqs = []
    for j, c in enumerate(cs):
        cam = cams[c]; f = fresh[c][0]
        sp = api.PixelSelector(f, 1, api.random_pattern(*cam.wh))
        sres, snum = sp.makeNewTracesBatch([0], [cam.ids[0]], [clouds[j]], [0.5 * dens[j]], [dens[j]], [1], cap=1 << 16)
        assert res[j][0].tobytes() == sres[0][0].tobytes() and res[j][1].tobytes() == sres[0][1].tobytes() and np.array_equal(num[j], snum[0]), c
        assert np.array_equal(ps.selectionMap(j), sp.selectionMap(0)) and len(res[j][0]) > 100, c
        T, onum, _ = orc.Selector(*cam.wh, api.random_pattern(*cam.wh)).makeNewTraces(cam.of[0], clouds[j], 0.5 * dens[j], dens[j], 1, np.zeros(cam.wh[::-1], np.float32))
        assert T.tobytes() == res[j][0].tobytes(), c
        K0, K1 = orc.distmap_geometry(cam.K, None, None); Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
        R, t = synth.rel_pose(cam.seq.R[0], cam.seq.t[0], cam.seq.R[3], cam.seq.t[3]); A = (K1 @ R.astype(np.float32) @ Ki0).astype(np.float32); B = (K1 @ t.astype(np.float32)).astype(np.float32)
        cl = cam.seq.clouds[1][::4]; uvid = np.stack([np.floor(cl[:, 0]), np.floor(cl[:, 1]), 1.0 / cl[:, 2]], 1).astype(np.float32)
        p = res[j][1]; cand4 = np.stack([p["u"], p["v"], rng.uniform(0.02, 0.3, len(p)), res[j][0]["my_type"]], 1).astype(np.float32)
        seqs.append(dict(pt_begin=[0, len(uvid)], KRKi=A[None], Kt=B[None], uvid=uvid, cand_begin=[0, len(cand4)], cKRKi=A[None], cKt=B[None], cand4=cand4, minActDist=2.0))
    decs, maps = api.activateSelectBatch(mixed, seqs, want_maps=True, cams=cs)
    for j, c in enumerate(cs):
        sdec, smaps = api.activateSelectBatch(fresh[c][0], [seqs[j]], want_maps=True)
        assert np.array_equal(decs[j], sdec[0]) and np.array_equal(maps[j], smaps[0]) and (decs[j] == 1).sum() > 10, c


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_change_nothing(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    L = api.LIB; c1 = cams[1]
    ctx = _mixed(api, synth, n_tracker_slots=4, max_frames=8, max_kf_images=8)
    for cam, lv in ((-1, 3), (8, 3), (1, 0), (1, 6), (1, -2)):
        assert L.sdv_set_camera_levels(ctx.p, cam, lv) == ERR_ARG, (cam, lv)
    assert L.sdv_set_camera_levels(None, 0, 0) == ERR_ARG
    ctx.makeImages(c1.ids[3], c1.seq.images[3], cam=1); ctx.makeImages(c1.ids[4], c1.seq.images[4], cam=1)
    ctx.setCalibSlots([1], [c1.K], cams=[1]); tr = api.CoarseTracker(ctx, 1); tr.setCoarseTrackingRef(c1.ids[3], c1.p4, c1.rh)
    clouds = [tr.cloud(l) for l in range(5)]
    assert L.sdv_set_camera_levels(ctx.p, 1, 4) == ERR_STATE                                  # a tracker reference built at 5 levels
    assert all(all(_same(x, y) for x, y in zip(a, tr.cloud(l))) for l, a in enumerate(clouds)) and tr.levels == 5
    # moving the slot to a camera of the same size and another depth
    ctx.setCameraSize(5, *SIZES[1]); ctx.setCameraLevels(5, 4)
    assert L.sdv_set_calib_slots_cams(ctx.p, 1, np.array([1], np.int32), api.C.addressof((api.sdv_calib * 1)(api.sdv_calib(*c1.K))), np.array([5], np.int32).ctypes.data) == ERR_STATE
    assert tr.levels == 5 and all(all(_same(x, y) for x, y in zip(a, tr.cloud(l))) for l, a in enumerate(clouds))
    ctx.setCameraLevels(5, 5); ctx.setCalibSlots([1], [c1.K], cams=[5]); ctx.setCalibSlots([1], [c1.K], cams=[1])     # same size and depth: allowed
    # a resident map alone blocks it too
    ctx.setCalibSlots([2], [c1.K], cams=[5]); rp = api.Reprojector(ctx); rp.setMap(2, [c1.ids[3], c1.ids[4]], c1.hT[:2], c1.hab[:2], c1.pts[c1.pts["host"] < 2])
    before = rp.reprojectMap(2, c1.ids[4], c1.poses[4])
    assert L.sdv_set_camera_levels(ctx.p, 5, 4) == ERR_STATE
    after = rp.reprojectMap(2, c1.ids[4], c1.poses[4])
    assert _same(before[0], after[0]) and _same(before[1], after[1]) and len(before[0]) > 5
    ctx._ck(L.sdv_map_clear(ctx.p, 2)); ctx.setCameraLevels(5, 4); ctx.setCameraLevels(5, 5)                  # without reference and map the depth may change
    # a coarsest level at or past a job's depth (or >= 5): nothing enqueued, poses untouched
    ctx.setCameraSize(6, 1200, 360); ctx.setCameraLevels(6, 4)
    T = np.stack([c1.Tgt, c1.Tgt]); ab = np.zeros((2, 2)); T0 = T.copy()
    for co in ([5, 2], [2, -1], [3, 5]):
        with pytest.raises(api.SdvError, match="error -1"):
            ctx.trackBatch([1, 1], [c1.ids[4]] * 2, T, ab, coarsest=co)
        assert _same(T, T0) and not ab.any()
    with pytest.raises(api.SdvError, match="error -1"):
        ctx.trackBatch([1], [c1.ids[4]], T[:1], ab[:1], coarsest=5)
    with pytest.raises(api.SdvError, match="error -1"):
        api.CoarseTracker(mixed, 8).calcRes(cams[4].ids[4], 3, _track_inits(cams[4], 1)[0], 0.0, 0.0, 20.0)
    r = mixed.trackBatch([8, 2], [cams[4].ids[4], c1.ids[4]], _track_inits(cams[4], 1).repeat(2, 0), np.zeros((2, 2)), coarsest=2)
    assert r["good"][0]
    T4 = np.stack([_track_inits(cams[4], 1)[0], c1.Tgt]); T40 = T4.copy()
    with pytest.raises(api.SdvError, match="error -1"):
        mixed.trackBatch([8, 2], [cams[4].ids[4], c1.ids[4]], T4, np.zeros((2, 2)), coarsest=3)    # level 3 is past camera 4's depth
    assert _same(T4, T40)
    # the selector's 3-level rule
    ctx.setCameraSize(7, 1200, 360); ctx.setCameraLevels(7, 2)
    ps = api.PixelSelector(ctx, 2, api.random_pattern(*CTX_WH), cams=[6, 0])
    with pytest.raises(api.SdvError, match="error -1"):
        ps.bindCams([0], [7])
    assert ps.slotSize(0) == (1200, 360)
    assert L.sdv_set_camera_levels(ctx.p, 6, 2) == ERR_STATE                                  # selector slot 0 is bound to camera 6
    ctx.setCameraLevels(6, 3); ps.bindCams([0], [0]); ctx.setCameraLevels(6, 2); ctx.setCameraLevels(6, 4)
    ctx.close()
    ctx0 = api.Context(_Ks(synth)[0], *CTX_WH, levels=CTX_L, max_frames=2); ctx0.setCameraLevels(0, 2)
    with pytest.raises(api.SdvError, match="error -1"):
        api.PixelSelector(ctx0, 1, api.random_pattern(*CTX_WH))
    ctx0.close()


# ------------------------------------------------------------------------------------------------ explicit context depth == never set
def test_explicit_context_depth_is_the_default():
    api, synth = _mods(); cam = Cam(synth, 1, _Ks(synth)[1])
    outs = []
    for explicit in (False, True):
        f = api.Context(cam.K, *cam.wh, levels=CTX_L, n_tracker_slots=2, max_frames=N + 2, max_kf_images=N + 2)
        if explicit:
            for c in range(8):
                f.setCameraLevels(c, CTX_L)
        rp = cam.load(api, f, [0, 1], 0)
        T = _track_inits(cam, 2); ab = np.zeros((2, 2)); r = f.trackBatch([0, 1], [cam.ids[4]] * 2, T, ab)
        order = np.random.default_rng(3).permutation(rp.n_cells).astype(np.int32)
        g = rp.refineBatch([0, 1], [cam.ids[5]] * 2, np.stack([cam.poses[5]] * 2), cell_order=order, max_matches=150)
        j = [dict(slot=0, frame=cam.ids[5], sprelast_c2w=cam.poses[3], slast_c2w=cam.poses[4], lastF_c2w=cam.poses[3], aff_last=[0.0, 0.0], poses_valid=1, lastCoarseRMSE=[1e-3] * 5)]
        tn = api.trackNewCoarseBatch(f, j, cell_order=order)[0]
        outs.append((T, ab, r, g, tn)); f.close()
    (Ta, aa, ra, ga, na), (Tb, ab_, rb, gb, nb) = outs
    assert _same(Ta, Tb) and _same(aa, ab_) and all(_same(ra[k], rb[k]) for k in ra) and all(_same(ga[k], gb[k]) for k in ("T", "n_matches", "res", "iterations", "accepts"))
    assert all(_same(na[k], nb[k]) for k in na) and (ra["iterations"][:, 4] > 0).all()
