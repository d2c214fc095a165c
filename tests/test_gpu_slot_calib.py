"""GPU tests (-m gpu) of per-slot intrinsics (sdv_set_calib_slots, CoarseTracker::makeK per tracker instance).

One context holds sequences of three cameras at 1200x360: slots 0-2 on the context calibration (camera A), slots 3-5 with camera B's K, slots 6-8
with a "BA-moved" K.  Every job of the mixed batch must give EXACTLY what the same job gives in a fresh context created with that slot's K, and each
camera's results must match the oracle run with that K (tolerances of test_gpu_tracker / _reproject / _refine / _policy)."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence

pytestmark = pytest.mark.gpu

N = 8                                                     # frames per camera
KFS = [0, 1, 2, 3]                                        # map keyframes; frame 3 is the tracking reference


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _cameras(synth):
    fx, fy, cx, cy = synth.KITTI_K
    return [tuple(synth.KITTI_K),
            (721.54, 721.54, 609.56 - 20.5, 172.85 - 8.0),          # another KITTI camera (sequence 03), same 1200x360 crop as synth.KITTI_K
            (fx * 1.01, fy * 0.99, cx + 2.0, cy - 2.0)]              # K after a bundle adjustment moved it


class Cam:
    """one camera: its rendered sequence (seed per camera: the sequence cache is keyed by seed and size only), map, reference cloud, oracle frames"""

    def __init__(self, api, synth, c, K):
        self.K = K; self.wh = synth.KITTI_WH; w, h = self.wh; self.L = api.pyr_levels(w, h)
        self.seq = seq = cached_sequence(N, 7101 + 101 * c, K, self.wh)
        self.ids = [1000 * (c + 1) + i for i in range(N)]
        self.pts, self.hT, self.hab = synth.make_map(seq, KFS, n_per_frame=400, seed=2)
        self.poses = np.array([np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(N)])
        ref = synth.select_points(seq.images[3], seq.clouds[3], 2000)
        self.p4 = np.concatenate([ref, np.full((len(ref), 1), 1e-3, np.float32)], 1).astype(np.float32); self.rh = np.zeros(len(self.p4), np.int32)
        self.frames = [orc.Frame(seq.images[i], self.L) for i in range(N)]
        self.Tgt = orc.se3_from_rt(*synth.rel_pose(seq.R[3], seq.t[3], seq.R[4], seq.t[4]))     # reference frame 3 -> tracked frame 4

    def load(self, api, ctx, slots):
        for i in range(N):
            ctx.makeImages(self.ids[i], self.seq.images[i])
        rp = api.Reprojector(ctx)
        for s in slots:
            api.CoarseTracker(ctx, s).setCoarseTrackingRef(self.ids[3], self.p4, self.rh)
            rp.setMap(s, [self.ids[k] for k in KFS], self.hT, self.hab, self.pts)
        return rp


def _contexts(api, synth, cams, **kw):
    """the mixed context (slot 3c+j -> camera c) and one fresh single-camera context per camera (slot j)"""
    w, h = synth.KITTI_WH
    mixed = api.Context(cams[0].K, w, h, n_tracker_slots=9, max_frames=3 * N + 2, **kw)
    mixed.setCalibSlots([3, 4, 5, 6, 7, 8], [cams[1].K] * 3 + [cams[2].K] * 3)
    mrp = [cam.load(api, mixed, [3 * c, 3 * c + 1, 3 * c + 2]) for c, cam in enumerate(cams)][0]
    fresh = []
    for cam in cams:
        f = api.Context(cam.K, w, h, n_tracker_slots=3, max_frames=N + 2, **kw); fresh.append((f, cam.load(api, f, [0, 1, 2])))
    return mixed, mrp, fresh


@pytest.fixture(scope="module")
def setup():
    api, synth = _mods()
    cams = [Cam(api, synth, c, K) for c, K in enumerate(_cameras(synth))]
    mixed, mrp, fresh = _contexts(api, synth, cams)
    yield api, synth, cams, mixed, mrp, fresh
    mixed.close()
    for f, _ in fresh:
        f.close()


def _track_inits(cam, k):
    """k initial guesses of the 3 -> 4 motion: from the true one to a few centimetres off (inside the tracker's basin)"""
    xis = ([0, 0, 0, 0, 0, 0], [0.01, -0.005, 0.02, 1e-3, -1e-3, 5e-4], [-0.03, 0.02, 0.04, -2e-3, 1e-3, 1e-3])
    return np.stack([orc.se3_mul(orc.se3_exp(xi), cam.Tgt) for xi in xis[:k]])


def _track_all(api, cams, mixed, fresh):
    """every slot of the mixed context in ONE launch vs each camera's three slots in its fresh context"""
    T = np.concatenate([_track_inits(cam, 3) for cam in cams]); ab = np.zeros((9, 2)); ab[1::3] = [0.02, 1.0]
    T0, ab0 = T.copy(), ab.copy()
    rm = mixed.trackBatch(list(range(9)), [cams[s // 3].ids[4] for s in range(9)], T, ab)
    for c, cam in enumerate(cams):
        Tf, abf = T0[3 * c:3 * c + 3].copy(), ab0[3 * c:3 * c + 3].copy()
        rf = fresh[c][0].trackBatch([0, 1, 2], [cam.ids[4]] * 3, Tf, abf)
        sl = slice(3 * c, 3 * c + 3)
        assert np.array_equal(T[sl], Tf) and np.array_equal(ab[sl], abf), c
        for key in ("good", "flow", "iterations", "accepts", "evals"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        assert np.array_equal(rm["lastResiduals"][sl], rf["lastResiduals"], equal_nan=True), c
    return T0, ab0, T, ab, rm


def test_calcres_and_gs_bit_equal_to_single_camera_context(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    for s in range(9):
        c, j = divmod(s, 3); cam = cams[c]
        T = _track_inits(cam, 2)[1]
        for l in range(cam.L):
            for cutoff, (a, b) in ((20.0, (0.0, 0.0)), (40.0, (0.03, -2.0))):
                rm = api.CoarseTracker(mixed, s).calcRes(cam.ids[4], l, T, a, b, cutoff); Hm, bm = api.CoarseTracker(mixed, s).calcGSSSE(l)
                rf = api.CoarseTracker(fresh[c][0], j).calcRes(cam.ids[4], l, T, a, b, cutoff); Hf, bf = api.CoarseTracker(fresh[c][0], j).calcGSSSE(l)
                assert np.array_equal(rm, rf, equal_nan=True) and np.array_equal(Hm, Hf, equal_nan=True) and np.array_equal(bm, bf, equal_nan=True), (s, l, cutoff)


def test_track_batch_bit_equal_and_matches_oracle_per_camera(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    T0, ab0, T, ab, rm = _track_all(api, cams, mixed, fresh)
    same = 0
    for s in range(9):
        cam = cams[s // 3]; w, h = cam.wh
        otr = orc.CoarseTracker(w, h, cam.L, cam.K); otr.setCoarseTrackingRef(cam.frames[3], cam.p4, cam.rh)
        ro = otr.trackNewestCoarse(cam.frames[4], T0[s], ab0[s], cam.L - 1)
        assert rm["good"][s] == ro["good"] and ro["good"], s
        e = np.abs(orc.se3_log(orc.se3_mul(T[s], orc.se3_inv(ro["T"])))).max()
        if np.array_equal(rm["iterations"][s], ro["iterations"]) and np.array_equal(rm["accepts"][s], ro["accepts"]):
            same += 1                                              # the same LM path: test_gpu_tracker's bounds
            assert np.array_equal(rm["evals"][s], ro["evals"]) and e < 1e-5 and np.allclose(ab[s], ro["ab"], atol=1e-3), s
            assert np.allclose(rm["lastResiduals"][s], ro["lastResiduals"], rtol=1e-4, equal_nan=True) and np.allclose(rm["flow"][s], ro["flow"], rtol=1e-3, atol=1e-6), s
        else:                                                      # an accept decision flipped on the last float bit (test_track_200_frame_pairs_vs_oracle)
            assert e < 5e-3, (s, e, rm["iterations"][s], ro["iterations"])
    assert same >= 8, same


@pytest.mark.parametrize("cfg", [dict(track_threads=64), dict(cluster_size=8, track_threads=256)])
def test_track_batch_bit_equal_other_launch_configs(setup, cfg):
    api, synth, cams = setup[:3]
    mixed, mrp, fresh = _contexts(api, synth, cams, **cfg)
    _track_all(api, cams, mixed, fresh)
    mixed.close()
    for f, _ in fresh:
        f.close()


def test_reproject_map_batch_bit_equal_and_matches_oracle(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    w, h = synth.KITTI_WH
    noisy = lambda T: np.concatenate([T[:4], T[4:] + [0.03, -0.01, 0.05]])
    jobs = []
    for s in range(9):
        cam = cams[s // 3]
        jobs += [dict(slot=s, cur=7, T=cam.poses[7], kf=-1, oh=-1, bk=0), dict(slot=s, cur=7, T=noisy(cam.poses[7]), kf=-1, oh=-1, bk=0)]
    jobs += [dict(slot=s, cur=0, T=cams[s // 3].poses[0], kf=0, oh=3, bk=1) for s in (1, 4, 7)]          # backprojectMap of one keyframe's points (only_host / backup)
    order = np.random.default_rng(4).permutation(mrp.n_cells).astype(np.int32)
    args = lambda js, idf: ([j["slot"] for j in js], [idf(j) for j in js], np.stack([j["T"] for j in js]), None, [j["kf"] for j in js], [j["oh"] for j in js], [j["bk"] for j in js])
    res = mrp.reprojectMapBatch(*args(jobs, lambda j: cams[j["slot"] // 3].ids[j["cur"]]), cell_order=order)
    for c, cam in enumerate(cams):
        mine = [k for k, j in enumerate(jobs) if j["slot"] // 3 == c]
        fj = [dict(jobs[k], slot=jobs[k]["slot"] % 3) for k in mine]
        rf = fresh[c][1].reprojectMapBatch(*args(fj, lambda j: cam.ids[j["cur"]]), cell_order=order)
        for k, g in zip(mine, rf):
            j = jobs[k]
            assert np.array_equal(res[k][0], g[0]) and np.array_equal(res[k][1], g[1]), (k, j)
            o = orc.reproject_map(w, h, cam.L, cam.K, [cam.frames[i] for i in KFS], cam.hT, cam.hab, cam.frames[j["cur"]], j["T"], [0.0, 0.0], cam.pts,
                                  cur_kf_index=j["kf"], only_host=j["oh"], backup=bool(j["bk"]), cell_order=order)
            assert len(o[0]) > 10 and np.array_equal(o[0], res[k][0]) and np.array_equal(o[1], res[k][1]), (k, j, len(o[0]), len(res[k][0]))


def test_refine_batch_bit_equal_and_matches_oracle(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    w, h = synth.KITTI_WH; rng = np.random.default_rng(3); order = rng.permutation(mrp.n_cells).astype(np.int32)
    T0 = np.stack([cams[s // 3].poses[7] + np.concatenate([np.zeros(4), rng.normal(0, 0.04, 3)]) for s in range(9)])
    rm = mrp.refineBatch(list(range(9)), [cams[s // 3].ids[7] for s in range(9)], T0, cell_order=order, max_matches=150)
    for c, cam in enumerate(cams):
        sl = slice(3 * c, 3 * c + 3)
        rf = fresh[c][1].refineBatch([0, 1, 2], [cam.ids[7]] * 3, T0[sl], cell_order=order, max_matches=150)
        for key in ("T", "n_matches", "res", "iterations", "accepts"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        for s in range(3 * c, 3 * c + 3):
            oi, opx = orc.reproject_map(w, h, cam.L, cam.K, [cam.frames[i] for i in KFS], cam.hT, cam.hab, cam.frames[7], T0[s], [0.0, 0.0], cam.pts, cell_order=order, max_matches=150)
            P = cam.pts
            p6 = np.stack([P["u"][oi], P["v"][oi], P["idepth"][oi], P["host"][oi].astype(np.float32), opx[:, 0].astype(np.float32), opx[:, 1].astype(np.float32)], 1).astype(np.float32)
            o = orc.struct_pose(w, h, np.array(cam.K, np.float32), cam.hT, p6, T0[s])
            assert rm["n_matches"][s] == len(oi) and (o["iterations"], o["accepts"]) == (int(rm["iterations"][s]), int(rm["accepts"][s])), s
            assert np.abs(o["T"] - rm["T"][s]).max() < 1e-9


def test_struct_pose_batch_slots_bit_equal_and_matches_oracle(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    w, h = synth.KITTI_WH
    ds = [synth.make_overlap_points(300 + 50 * s, 2 + s % 4, 40 + s, K=cams[s // 3].K, outlier_frac=0.05) for s in range(9)]
    T = np.stack([d["T_init"] for d in ds])
    rm = api.structPoseEstimationBatch(mixed, T.copy(), [d["pts"] for d in ds], [d["host_T7"] for d in ds], slots=list(range(9)))
    for c, cam in enumerate(cams):
        sl = slice(3 * c, 3 * c + 3)
        rf = api.structPoseEstimationBatch(fresh[c][0], T[sl].copy(), [d["pts"] for d in ds[sl]], [d["host_T7"] for d in ds[sl]])
        for key in ("T", "res", "iterations", "accepts"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        for s in range(3 * c, 3 * c + 3):
            p = ds[s]["pts"]; p6 = np.stack([p["u"], p["v"], p["idepth"], p["host"].astype(np.float32), p["obs_x"], p["obs_y"]], 1).astype(np.float32)
            o = orc.struct_pose(w, h, np.array(cam.K, np.float32), ds[s]["host_T7"], p6, T[s])
            assert (int(rm["iterations"][s]), int(rm["accepts"][s])) == (o["iterations"], o["accepts"]) and np.abs(rm["T"][s] - o["T"]).max() < 1e-9, s
    # CoarseTracker.structPoseEstimation uses its own slot's K
    g = api.CoarseTracker(mixed, 7).structPoseEstimation(T[7], ds[7]["pts"], ds[7]["host_T7"])
    assert np.array_equal(g["T"], rm["T"][7]) and g["iterations"] == rm["iterations"][7]


def test_track_new_coarse_batch_bit_equal_and_matches_oracle(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    order = np.random.default_rng(4).permutation(mrp.n_cells).astype(np.int32)

    def jobs_of(cam, slots):
        P = cam.poses; base = dict(frame=cam.ids[6], sprelast_c2w=P[4], slast_c2w=P[5], lastF_c2w=P[3], aff_last=[0.0, 0.0])
        return [dict(base, slot=slots[0], poses_valid=1, lastCoarseRMSE=[100.0] * 5),                          # healthy: one try
                dict(base, slot=slots[1], poses_valid=1, lastCoarseRMSE=[1e-3] * 5),                           # all 31 hypotheses
                dict(base, slot=slots[2], poses_valid=0, lastCoarseRMSE=[100.0] * 5, frame=cam.ids[4])]        # invalid history: identity only
    jm = sum([jobs_of(cam, [3 * c, 3 * c + 1, 3 * c + 2]) for c, cam in enumerate(cams)], [])
    rm = api.trackNewCoarseBatch(mixed, jm, cell_order=order)
    for c, cam in enumerate(cams):
        jf = jobs_of(cam, [0, 1, 2]); rf = api.trackNewCoarseBatch(fresh[c][0], jf, cell_order=order)
        w, h = cam.wh; otr = orc.CoarseTracker(w, h, cam.L, cam.K); otr.setCoarseTrackingRef(cam.frames[3], cam.p4, cam.rh)
        for k, (j, g) in enumerate(zip(jf, rf)):
            m = rm[3 * c + k]
            for key in g:
                assert np.array_equal(np.asarray(m[key]), np.asarray(g[key]), equal_nan=True), (c, k, key)
            o = orc.track_new_coarse(otr, cam.frames[cam.ids.index(j["frame"])], cam.K, [cam.frames[i] for i in KFS], cam.hT, cam.hab, cam.pts, j["sprelast_c2w"], j["slast_c2w"],
                                     j["lastF_c2w"], j["aff_last"], j["poses_valid"], j["lastCoarseRMSE"], cell_order=order)
            assert m["tries"] == o["tries"] and m["have_one_good"] == o["have_one_good"], (c, k, m["tries"], o["tries"])
            assert np.allclose(m["lastCoarseRMSE"], o["lastCoarseRMSE"], rtol=1e-4, equal_nan=True) and np.allclose(m["aff_g2l"], o["aff_g2l"], atol=2e-4)
            # the tracker's float sums run in another order than the oracle's, so an LM accept decision can flip (test_track_200_frame_pairs_vs_oracle), here on
            # the 31-hypothesis job of camera A, which runs on the context calibration; structPoseEstimation compares float energies too and can then take
            # another accept path from the tracked pose.  Same tries, winner and match count; poses within north_star's bound.
            assert m["n_matches"] == o["n_matches"], (c, k, m["n_matches"], o["n_matches"])
            assert np.abs(m["camToTrackingRef"] - o["camToTrackingRef"]).max() < 1e-3 and np.abs(m["camToWorld"] - o["camToWorld"]).max() < 1e-3, (c, k)
        assert [r["tries"] for r in rf] == [1, 31, 1]


def test_semantics_default_own_clear_and_rejected_calls(setup):
    api, synth, cams = setup[:3]
    KA, KB, KC = (cam.K for cam in cams); cam = cams[0]; w, h = cam.wh
    ctx = api.Context(KB, w, h, n_tracker_slots=3, max_frames=N + 2); rp = cam.load(api, ctx, [0, 1, 2])
    ref = {K: api.Context(K, w, h, n_tracker_slots=1, max_frames=N + 2) for K in (KA, KB, KC)}
    refrp = {K: cam.load(api, r, [0]) for K, r in ref.items()}
    T = _track_inits(cam, 2)[1]

    def calc(cx, slot):
        tr = api.CoarseTracker(cx, slot); out = []
        for l in range(cam.L):
            out.append(tr.calcRes(cam.ids[4], l, T, 0.0, 0.0, 20.0)); out.append(tr.calcGSSSE(l)[0])
        return np.concatenate([np.ravel(x) for x in out])

    def reproj(cx_rp, slot):
        return cx_rp.reprojectMap(slot, cam.ids[7], cam.poses[7])

    def same(a, b):
        return np.array_equal(a, b, equal_nan=True)
    want = {K: calc(r, 0) for K, r in ref.items()}; want_rp = {K: reproj(refrp[K], 0) for K in ref}
    assert not same(want[KA], want[KC]) and not same(want_rp[KA][1], want_rp[KC][1])
    assert same(calc(ctx, 0), want[KB])                                                 # no own K: the context calibration
    ctx.setCalib(KA); assert same(calc(ctx, 0), want[KA])                               # ... and it follows setCalib
    api.CoarseTracker(ctx, 1).makeK(KC)
    assert same(calc(ctx, 1), want[KC]) and same(calc(ctx, 0), want[KA])
    ctx.setCalib(KB); assert same(calc(ctx, 1), want[KC]) and same(calc(ctx, 0), want[KB])                                # own K kept across setCalib
    api.CoarseTracker(ctx, 1).setCoarseTrackingRef(cam.ids[3], cam.p4, cam.rh); assert same(calc(ctx, 1), want[KC])      # ... a new reference
    rp.setMap(1, [cam.ids[k] for k in KFS], cam.hT, cam.hab, cam.pts); g = reproj(rp, 1)                                 # ... and a new map
    assert same(g[0], want_rp[KC][0]) and same(g[1], want_rp[KC][1])
    # rejected calls change nothing: a bad slot, fx <= 0, NaNs, each in the middle of an otherwise valid list
    for slots, Ks in (([0, 9, 2], [KA, KA, KA]), ([0, -1, 2], [KA, KA, KA]), ([0, 1, 2], [KA, (0.0, 700.0, 600.0, 180.0), KA]),
                      ([0, 1, 2], [KA, (np.nan, 700.0, 600.0, 180.0), KA]), ([0, 1, 2], [KA, (700.0, 700.0, np.nan, 180.0), KA]),
                      ([0, 1, 2], [KA, (700.0, np.inf, 600.0, 180.0), KA])):
        with pytest.raises(api.SdvError):
            ctx.setCalibSlots(slots, Ks)
    with pytest.raises(api.SdvError):
        ctx.clearCalibSlots([0, 3])
    assert same(calc(ctx, 0), want[KB]) and same(calc(ctx, 1), want[KC]) and same(calc(ctx, 2), want[KB])
    g = reproj(rp, 1); assert same(g[0], want_rp[KC][0]) and same(g[1], want_rp[KC][1])
    ctx.clearCalibSlots([1]); assert same(calc(ctx, 1), want[KB])                      # back to the context calibration
    g = reproj(rp, 1); assert same(g[0], want_rp[KB][0]) and same(g[1], want_rp[KB][1])
    # coarseTracker / coarseTracker_forNewKF: two slots of one sequence, same reference, different K, one launch, independent
    ctx.setCalib(KA); api.CoarseTracker(ctx, 1).makeK(KC)
    Tm = np.stack([T, T]); abm = np.zeros((2, 2)); rm = ctx.trackBatch([0, 1], [cam.ids[4]] * 2, Tm, abm)
    for k, K in enumerate((KA, KC)):
        Tr = T[None].copy(); abr = np.zeros((1, 2)); rr = ref[K].trackBatch([0], [cam.ids[4]], Tr, abr)
        assert np.array_equal(Tm[k], Tr[0]) and np.array_equal(abm[k], abr[0]) and np.array_equal(rm["iterations"][k], rr["iterations"][0]), K
    assert not np.array_equal(Tm[0], Tm[1])
    ctx.close()
    for r in ref.values():
        r.close()
