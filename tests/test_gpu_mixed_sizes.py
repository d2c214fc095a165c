"""GPU tests (-m gpu) of cameras of different rectified sizes in one context (sdv_set_camera_size and the _cams entries).

The context has KITTI-360's size, 1400x360, on camera 0.  Camera 1 is KITTI 00 (1200x360); camera 2 is 1244x356 at the context's 4 levels, whose level 2
is 311 wide (the odd-intermediate pyramid path).  In every check the per-size reference is a fresh context created at that frame's own size: every frame
and every job of a mixed batch must give exactly what it gives there, and the pyramids must equal the oracle's makeImages."""
import ctypes as C
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from test_undistort import CALIBS, _check_levels, _mirror

pytestmark = pytest.mark.gpu

SIZES = [(1400, 360), (1200, 360), (1244, 356), (1202, 360)]   # camera c's rectified size; 1202 % 4 == 2: a batch with camera 3 takes the scalar pyramid path
LEVELS = 4                                                 # pyr_levels(1400, 360) == pyr_levels(1200, 360) == 4
N = 8                                                      # frames per camera
KFS = [0, 1, 2, 3]                                         # map keyframes; frame 3 is the tracking reference
ERR_ARG, ERR_STATE = -1, -5


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _Ks(synth):
    return [tuple(synth.K360_K), tuple(synth.KITTI_K), (702.5, 698.0, 611.0, 171.5), (700.0, 700.0, 600.5, 175.0)]


def _mixed(api, synth, levels=LEVELS, **kw):
    ctx = api.Context(synth.K360_K, *SIZES[0], levels=levels, **kw)
    for c in (1, 2, 3):
        ctx.setCameraSize(c, *SIZES[c])
    return ctx


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _levels(ctx, fid, L):
    return [ctx.frameLevel(fid, l) for l in range(L)]


def _same_levels(a, b):
    return all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(a, b))


def filtered_order(order, c):
    """the context grid's cell_order as camera c's job walks it (sdv_b200.h, sdv_reproject_map_batch): cells outside its grid skipped, its own numbering"""
    ncols = -(-SIZES[0][0] // 25); jc, jr = -(-SIZES[c][0] // 25), -(-SIZES[c][1] // 25)
    return np.array([(k // ncols) * jc + k % ncols for k in order if k % ncols < jc and k // ncols < jr], np.int32)


# ------------------------------------------------------------------------------------------------ ingest
MIX = [0, 1, 2, 2, 0, 1, 1, 2, 0]                          # camera of each frame of a mixed batch: every width % 4 == 0 (16-byte vector path)
MIX_W2 = [3, 0, 1, 3, 2, 0, 3, 1, 2]                       # with a 1202-wide camera: the whole batch takes the scalar path
RAW_MIX = [0, 1, 1, 0, 1, 0]                               # raw: KITTI-360 tables on camera 0, KITTI 00 tables on camera 1


def _images(mix, seed):
    rng = np.random.default_rng(seed); out = []
    for k, c in enumerate(mix):
        w, h = SIZES[c]
        if k % 2:
            out.append(rng.integers(0, 256, (h, w)).astype(np.uint8))
        else:
            yy, xx = np.mgrid[0:h, 0:w]; out.append(((xx * 3 + yy * 5 + 7 * k) % 256).astype(np.uint8))
    return out


def _ingest(api, ctx, ids, imgs8, fmt, cams, keep):
    """one batch of imgs8 (mono8 host arrays) in format fmt; returns the float images the frames must hold"""
    import torch
    f32 = [np.ascontiguousarray(i.astype(np.float32)) for i in imgs8]
    if fmt == "host_f32":
        ctx.makeImagesBatch(ids, [a.ctypes.data for a in f32], cams=cams)
    elif fmt == "host_u8":
        ctx.makeImagesBatch(ids, [a.ctypes.data for a in imgs8], u8=True, cams=cams)
    elif fmt in ("dev_f32", "dev_u8", "adopt"):
        ts = [torch.from_numpy(a if fmt == "dev_u8" else b).cuda() for a, b in zip(imgs8, f32)]; torch.cuda.synchronize(); keep.extend(ts)
        ctx.makeImagesBatch(ids, [t.data_ptr() for t in ts], device=True, u8=fmt == "dev_u8", adopt=fmt == "adopt", cams=cams)
    ctx.sync()
    return f32


FORMATS = ["host_f32", "host_u8", "dev_f32", "dev_u8", "adopt"]


def _check_ingest(levels):
    api, synth = _mods(); Ks = _Ks(synth)
    unds = [_mirror(CALIBS["kitti360"]), _mirror(CALIBS["kitti00"])]
    ctx = _mixed(api, synth, levels, max_frames=112, max_kf_images=112); L = ctx.levels
    singles = [api.Context(Ks[c], *SIZES[c], levels=L, max_frames=48, max_kf_images=48) for c in range(4)]
    for c in (0, 1):
        ctx.setUndistort(unds[c], cam=c); singles[c].setUndistort(unds[c])
    keep = []; fid = 0; got = {}
    for i, (fmt, mix) in enumerate([(f, m) for m in (MIX, MIX_W2) for f in FORMATS]):
        imgs8 = _images(mix, 30 + i); ids = list(range(fid, fid + len(mix))); fid += len(mix)
        want = _ingest(api, ctx, ids, imgs8, fmt, mix, keep)
        for k, c in enumerate(mix):
            _check_levels(api, ctx, ids[k], want[k], L)                                                   # the oracle's makeImages
            _ingest(api, singles[c], [ids[k]], [imgs8[k]], fmt, None, keep)                                  # the unchanged single-size entries
            got[ids[k]] = _levels(ctx, ids[k], L)
            assert _same_levels(got[ids[k]], _levels(singles[c], ids[k], L)), (fmt, k, c)
    rng = np.random.default_rng(5)
    raws = [rng.integers(0, 256, (unds[c].hOrg, unds[c].wOrg)).astype(np.uint8) for c in RAW_MIX]
    ids = list(range(fid, fid + len(RAW_MIX)))
    ctx.makeImagesBatch(ids, [r.ctypes.data for r in raws], raw=True, cams=RAW_MIX); ctx.sync()
    for k, c in enumerate(RAW_MIX):
        _check_levels(api, ctx, ids[k], unds[c].undistort_host(raws[k]), L)
        singles[c].makeImagesRaw(ids[k], raws[k])
        assert _same_levels(_levels(ctx, ids[k], L), _levels(singles[c], ids[k], L)), ("raw", k, c)
    # re-ingest the first batch's handles with new content (packed-texel cache dropped and rebuilt at each frame's size), cameras permuted
    ids = list(range(len(MIX))); mix2 = MIX[3:] + MIX[:3]; imgs8 = _images(mix2, 99)
    want = _ingest(api, ctx, ids, imgs8, "host_f32", mix2, keep)
    for k in range(len(ids)):
        _check_levels(api, ctx, ids[k], want[k], L)
    ctx.close()
    for s in singles:
        s.close()


def test_mixed_ingest_every_format_bit_exact():
    _check_ingest(LEVELS)


def test_mixed_ingest_single_level_context():
    """levels == 1: pyr_copy0_kernel / pyr_remap0_kernel at each frame's size"""
    _check_ingest(1)


# ------------------------------------------------------------------------------------------------ per-frame path
class Cam:
    """one camera size: its rendered sequence, map, reference cloud"""

    def __init__(self, api, synth, c, K):
        self.c, self.K, self.wh = c, K, SIZES[c]
        self.seq = seq = cached_sequence(N, 7301 + 101 * c, K, self.wh)
        self.ids = [1000 * (c + 1) + i for i in range(N)]
        self.pts, self.hT, self.hab = synth.make_map(seq, KFS, n_per_frame=400, seed=2)
        self.poses = np.array([np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(N)])
        ref = synth.select_points(seq.images[3], seq.clouds[3], 2000)
        self.p4 = np.concatenate([ref, np.full((len(ref), 1), 1e-3, np.float32)], 1).astype(np.float32); self.rh = np.zeros(len(self.p4), np.int32)
        self.Tgt = orc.se3_from_rt(*synth.rel_pose(seq.R[3], seq.t[3], seq.R[4], seq.t[4]))

    def load(self, api, ctx, slots, cam):
        for i in range(N):
            ctx.makeImages(self.ids[i], self.seq.images[i], cam=cam)
        rp = api.Reprojector(ctx)
        for s in slots:
            api.CoarseTracker(ctx, s).setCoarseTrackingRef(self.ids[3], self.p4, self.rh)
            rp.setMap(s, [self.ids[k] for k in KFS], self.hT, self.hab, self.pts)
        return rp


def _contexts(api, synth, cams, **kw):
    """the mixed context (slot 3c+j -> camera c; camera 0 on the context calibration) and one fresh context per size (slot j)"""
    mixed = _mixed(api, synth, n_tracker_slots=9, max_frames=3 * N + 2, max_kf_images=3 * N + 2, **kw)
    mixed.setCalibSlots([3, 4, 5, 6, 7, 8], [cams[1].K] * 3 + [cams[2].K] * 3, cams=[1, 1, 1, 2, 2, 2])
    mrp = [cam.load(api, mixed, [3 * c, 3 * c + 1, 3 * c + 2], c) for c, cam in enumerate(cams)][0]
    fresh = []
    for cam in cams:
        f = api.Context(cam.K, *cam.wh, levels=LEVELS, n_tracker_slots=3, max_frames=N + 2, max_kf_images=N + 2, **kw); fresh.append((f, cam.load(api, f, [0, 1, 2], 0)))
    return mixed, mrp, fresh


@pytest.fixture(scope="module")
def setup():
    api, synth = _mods()
    cams = [Cam(api, synth, c, K) for c, K in enumerate(_Ks(synth)[:3])]
    mixed, mrp, fresh = _contexts(api, synth, cams)
    yield api, synth, cams, mixed, mrp, fresh
    mixed.close()
    for f, _ in fresh:
        f.close()


def _track_inits(cam, k):
    xis = ([0, 0, 0, 0, 0, 0], [0.01, -0.005, 0.02, 1e-3, -1e-3, 5e-4], [-0.03, 0.02, 0.04, -2e-3, 1e-3, 1e-3])
    return np.stack([orc.se3_mul(orc.se3_exp(xi), cam.Tgt) for xi in xis[:k]])


def _track_all(api, cams, mixed, fresh):
    """every slot of the mixed context in ONE launch vs each size's three slots in its fresh context"""
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
        assert _same(rm["lastResiduals"][sl], rf["lastResiduals"]), c
        assert (rf["evals"][:, 0] > 0).all() and rf["good"].all(), c


def test_coarse_depth_clouds_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    for s in range(9):
        c, j = divmod(s, 3)
        for l in range(LEVELS):
            a, b = api.CoarseTracker(mixed, s).cloud(l), api.CoarseTracker(fresh[c][0], j).cloud(l)
            assert len(a[0]) > 0 and all(_same(x, y) for x, y in zip(a, b)), (s, l)


def test_calcres_and_gs_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    for s in range(9):
        c, j = divmod(s, 3); cam = cams[c]; T = _track_inits(cam, 2)[1]
        for l in range(LEVELS):
            for cutoff, (a, b) in ((20.0, (0.0, 0.0)), (40.0, (0.03, -2.0))):
                tm, tf = api.CoarseTracker(mixed, s), api.CoarseTracker(fresh[c][0], j)
                rm = tm.calcRes(cam.ids[4], l, T, a, b, cutoff); Hm, bm = tm.calcGSSSE(l)
                rf = tf.calcRes(cam.ids[4], l, T, a, b, cutoff); Hf, bf = tf.calcGSSSE(l)
                assert _same(rm, rf) and _same(Hm, Hf) and _same(bm, bf), (s, l, cutoff)


def test_track_batch_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    _track_all(api, cams, mixed, fresh)


def test_track_batch_bit_equal_cluster_launch(setup):
    api, synth, cams = setup[:3]
    mixed, mrp, fresh = _contexts(api, synth, cams, cluster_size=8, track_threads=256)
    _track_all(api, cams, mixed, fresh)
    mixed.close()
    for f, _ in fresh:
        f.close()


def test_track_new_coarse_batch_bit_equal(setup):
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
        rf = api.trackNewCoarseBatch(fresh[c][0], jobs_of(cam, [0, 1, 2]), cell_order=filtered_order(order, c))
        for k, g in enumerate(rf):
            for key in g:
                assert _same(rm[3 * c + k][key], g[key]), (c, k, key)
        assert [r["tries"] for r in rf] == [1, 31, 1] and all(r["n_matches"] > 10 for r in rf), c


def test_reproject_map_batch_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    noisy = lambda T: np.concatenate([T[:4], T[4:] + [0.03, -0.01, 0.05]])
    jobs = []
    for s in (4, 0, 7, 1, 5, 8, 2, 3, 6):                                                                     # cameras interleaved in the batch
        cam = cams[s // 3]
        jobs += [dict(slot=s, cur=7, T=cam.poses[7], kf=-1, oh=-1, bk=0), dict(slot=s, cur=7, T=noisy(cam.poses[7]), kf=-1, oh=-1, bk=0)]
    jobs += [dict(slot=s, cur=0, T=cams[s // 3].poses[0], kf=0, oh=3, bk=1) for s in (7, 1, 4)]              # backprojectMap of one keyframe's points (only_host / backup)
    order = np.random.default_rng(9).permutation(mrp.n_cells).astype(np.int32)
    args = lambda js, idf: ([j["slot"] for j in js], [idf(j) for j in js], np.stack([j["T"] for j in js]), None, [j["kf"] for j in js], [j["oh"] for j in js], [j["bk"] for j in js])
    res = mrp.reprojectMapBatch(*args(jobs, lambda j: cams[j["slot"] // 3].ids[j["cur"]]), cell_order=order, max_matches=250)
    for c, cam in enumerate(cams):
        mine = [k for k, j in enumerate(jobs) if j["slot"] // 3 == c]
        fj = [dict(jobs[k], slot=jobs[k]["slot"] % 3) for k in mine]
        rf = fresh[c][1].reprojectMapBatch(*args(fj, lambda j: cam.ids[j["cur"]]), cell_order=filtered_order(order, c), max_matches=250)
        for k, g in zip(mine, rf):
            assert len(g[0]) > 10 and _same(res[k][0], g[0]) and _same(res[k][1], g[1]), (k, jobs[k]["slot"])
    # all jobs on camera 0: the context order itself, identical to the fresh 1400x360 context
    r0 = mrp.reprojectMapBatch([0, 1], [cams[0].ids[7]] * 2, np.stack([cams[0].poses[7]] * 2), cell_order=order)
    f0 = fresh[0][1].reprojectMapBatch([0, 1], [cams[0].ids[7]] * 2, np.stack([cams[0].poses[7]] * 2), cell_order=order)
    assert all(_same(a[0], b[0]) and _same(a[1], b[1]) for a, b in zip(r0, f0))


def test_refine_batch_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    rng = np.random.default_rng(3); order = rng.permutation(mrp.n_cells).astype(np.int32)
    T0 = np.stack([cams[s // 3].poses[7] + np.concatenate([np.zeros(4), rng.normal(0, 0.04, 3)]) for s in range(9)])
    rm = mrp.refineBatch(list(range(9)), [cams[s // 3].ids[7] for s in range(9)], T0, cell_order=order, max_matches=150)
    for c, cam in enumerate(cams):
        sl = slice(3 * c, 3 * c + 3)
        rf = fresh[c][1].refineBatch([0, 1, 2], [cam.ids[7]] * 3, T0[sl], cell_order=filtered_order(order, c), max_matches=150)
        for key in ("T", "n_matches", "res", "iterations", "accepts"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        assert (rf["n_matches"] > 10).all(), c


def test_struct_pose_batch_slots_bit_equal(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    ds = [synth.make_overlap_points(300 + 50 * s, 2 + s % 4, 40 + s, K=cams[s // 3].K, wh=cams[s // 3].wh, outlier_frac=0.05) for s in range(9)]
    T = np.stack([d["T_init"] for d in ds])
    rm = api.structPoseEstimationBatch(mixed, T.copy(), [d["pts"] for d in ds], [d["host_T7"] for d in ds], slots=list(range(9)))
    for c in range(3):
        sl = slice(3 * c, 3 * c + 3)
        rf = api.structPoseEstimationBatch(fresh[c][0], T[sl].copy(), [d["pts"] for d in ds[sl]], [d["host_T7"] for d in ds[sl]], slots=[0, 1, 2])
        for key in ("T", "res", "iterations", "accepts"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)


def test_make_k_on_camera1_slot_then_track_and_refine(setup):
    """CoarseTracker::makeK at a keyframe on a KITTI slot of the mixed context keeps the slot on its camera: tracking and refinement afterwards are bit-identical
    to a 1200x360 context given the same makeK.  sdv_set_calib_slots (camera 0) on a slot that holds a reference or a map is refused and changes nothing."""
    api, synth, cams = setup[:3]
    cam = cams[1]; K2 = (cam.K[0] * 1.01, cam.K[1] * 0.99, cam.K[2] + 2.0, cam.K[3] - 2.0)
    mixed = _mixed(api, synth, n_tracker_slots=3, max_frames=N + 2, max_kf_images=N + 2)
    mixed.setCalibSlots([0, 1, 2], [cam.K] * 3, cams=[1] * 3); mrp = cam.load(api, mixed, [0, 1], 1)
    mrp.setMap(2, [cam.ids[k] for k in KFS], cam.hT, cam.hab, cam.pts)                           # slot 2: a map, no tracker reference
    one = api.Context(cam.K, *cam.wh, levels=LEVELS, n_tracker_slots=2, max_frames=N + 2, max_kf_images=N + 2); orp = cam.load(api, one, [0, 1], 0)
    T = _track_inits(cam, 2)[1][None]; order = np.random.default_rng(6).permutation(mrp.n_cells).astype(np.int32)

    def track_refine(ctx, rp, slot, co):
        Tt, ab = T.copy(), np.zeros((1, 2)); r = ctx.trackBatch([slot], [cam.ids[4]], Tt, ab)
        f = rp.refineBatch([slot], [cam.ids[7]], cam.poses[7][None], cell_order=co, max_matches=150)
        return Tt, ab, r, f
    before = track_refine(mixed, mrp, 1, order)
    for s in (1, 2):                                                                               # would move the slot back to camera 0
        kk = (api.sdv_calib * 1)(api.sdv_calib(*map(float, K2)))
        assert api.LIB.sdv_set_calib_slots(mixed.p, 1, np.array([s], np.int32), C.addressof(kk)) == ERR_STATE, s
    again = track_refine(mixed, mrp, 1, order)
    assert all(_same(a, b) for a, b in zip(before[:2], again[:2])) and _same(before[3]["T"], again[3]["T"])
    for ctx, rp, co in ((mixed, mrp, order), (one, orp, filtered_order(order, 1))):
        tr = api.CoarseTracker(ctx, 0); tr.makeK(K2); tr.setCoarseTrackingRef(cam.ids[3], cam.p4, cam.rh)    # setCoarseTrackingRef after makeK, as at a keyframe
        rp.setMap(0, [cam.ids[k] for k in KFS], cam.hT, cam.hab, cam.pts)
    assert mixed.slot_cam[0] == 1
    gm, go = track_refine(mixed, mrp, 0, order), track_refine(one, orp, 0, filtered_order(order, 1))
    assert _same(gm[0], go[0]) and _same(gm[1], go[1]) and gm[2]["good"][0] and np.array_equal(gm[2]["iterations"], go[2]["iterations"])
    for key in ("T", "n_matches", "res", "iterations", "accepts"):
        assert np.array_equal(gm[3][key], go[3][key]), key
    assert gm[3]["n_matches"][0] > 10 and not _same(gm[0], before[0])                                # the moved K was used
    mixed._ck(api.LIB.sdv_map_clear(mixed.p, 2)); mixed.setCalibSlots([2], [K2])                               # once the map is gone the slot may move
    mixed.close(); one.close()


# ------------------------------------------------------------------------------------------------ back end
def test_optimize_batch_and_marginalisation_bit_equal():
    """one 1200-wide and one 1400-wide window optimised in one device-resident schedule, then the keyframe hand-over, against each window alone in a context of its size"""
    api, synth = _mods(); Ks = _Ks(synth)
    seqs = {c: cached_sequence(8, 2000 + c, Ks[c], SIZES[c]) for c in (1, 0)}
    kfs = {1: [0, 1, 2, 3, 4, 5, 6], 0: [1, 2, 4, 5, 7]}
    wins = {c: synth.make_ba_window(seqs[c], kfs[c], n_per_frame=180, seed=20 + c, pose_noise=(0.005, 0.0003), match_noise=0.2, prior_scale=1e-3) for c in (1, 0)}
    mixed = _mixed(api, synth, max_frames=20, max_kf_images=20)
    ids = {c: [100 * (c + 1) + k for k in kfs[c]] for c in (1, 0)}
    for c in (1, 0):
        for k, f in zip(kfs[c], ids[c]):
            mixed.makeImages(f, seqs[c].images[k], cam=c)
    gbs = [api.EnergyFunctional(mixed, wins[c], ids[c], window=i) for i, c in enumerate((1, 0))]
    r = api.optimize_batch(mixed, [0, 1], 6)
    for i, c in enumerate((1, 0)):
        one = api.Context(Ks[c], *SIZES[c], max_frames=10, max_kf_images=10)
        for k, f in zip(kfs[c], ids[c]):
            one.makeImages(f, seqs[c].images[k])
        gb1 = api.EnergyFunctional(one, wins[c], ids[c]); r1 = api.optimize_batch(one, [0], 6)
        assert (r["iterations"][i], r["accepts"][i], r["rmse"][i]) == (r1["iterations"][0], r1["accepts"][0], r1["rmse"][0]) and r1["accepts"][0] > 0, c
        gb = gbs[i]; fa, fb = gb.frames(), gb1.frames()
        assert _same(fa["T_eval"], fb["T_eval"]) and _same(fa["state"], fb["state"]) and _same(gb.points()["idepth"], gb1.points()["idepth"]), c
        sel = (wins[c]["host"] == 1).astype(np.int32); sel[::4] = 1; sel[wins[c]["host"] == wins[c]["nF"] - 1] = 0
        sa, sb = gb.flagPointsForRemoval(sel), gb1.flagPointsForRemoval(sel)
        assert _same(sa, sb) and (sa == 2).sum() > 0
        ma, mb = gb.marginalizePointsF(), gb1.marginalizePointsF()
        assert all(_same(ma[k], mb[k]) for k in ("M", "Mb", "Msc", "Mbsc")), c
        gb.marginalizeFrame(1); gb1.marginalizeFrame(1)
        assert all(_same(x, y) for x, y in zip(gb.prior(), gb1.prior())), c
        one.close()
    mixed.close()


# ------------------------------------------------------------------------------------------------ refusals
def _lib_level0_pixels(api, ctx, img, cam, fid):
    """level-0 pixels the library holds for frame fid (ingested first from img on camera cam when img is given), read into an oversized sentinel buffer:
    the library's own idea of the camera's size, not the api's"""
    W, H = SIZES[0]
    if img is not None:
        src = np.zeros(W * H, np.float32); src[:img.size] = img.reshape(-1)            # room for any size a refused call might have left behind
        ctx.makeImagesBatch([fid], [src.ctypes.data], cams=[cam]); ctx.sync()
    buf = np.full(3 * (W * H + 4096), -7777.0, np.float32)
    ctx._ck(api.LIB.sdv_frame_download(ctx.p, fid, 0, buf.ctypes.data, None))
    return (int(np.nonzero(buf != -7777.0)[0].max()) + 1) // 3


def test_refusals_change_nothing(setup):
    api, synth, cams, mixed, mrp, fresh = setup
    L = api.LIB
    ctx = _mixed(api, synth, n_tracker_slots=4, max_frames=12, max_kf_images=12)
    for cam, wh in ((1, (1402, 360)), (1, (1400, 362)), (0, (1200, 360)), (8, (1200, 360)), (-1, (1200, 360)), (1, (1201, 360)), (1, (6, 360)), (1, (0, 360))):
        assert L.sdv_set_camera_size(ctx.p, cam, *wh) == ERR_ARG, (cam, wh)                     # larger than the context, camera 0, out of range, odd, empty level
    assert _lib_level0_pixels(api, ctx, cams[1].seq.images[0], 1, 9) == SIZES[1][0] * SIZES[1][1]   # the library's camera 1 is still 1200x360
    u = _mirror(CALIBS["kitti00"])
    ctx.setUndistort(u, cam=1)
    assert L.sdv_set_camera_size(ctx.p, 1, 1000, 300) == ERR_STATE                               # tables of the current size
    ctx.makeImages(7, cams[2].seq.images[0], cam=2)
    assert L.sdv_set_camera_size(ctx.p, 2, 1000, 300) == ERR_STATE                               # a resident frame
    assert _lib_level0_pixels(api, ctx, None, 2, 7) == SIZES[2][0] * SIZES[2][1]
    ctx.releaseFrame(7); ctx.setCameraSize(2, 1000, 300); ctx.setCameraSize(2, *SIZES[2])
    ctx.setCameraSize(3, 1000, 300); ctx.setCalibSlots([3], [cams[1].K], cams=[3])
    assert L.sdv_set_camera_size(ctx.p, 3, 1200, 360) == ERR_STATE                               # a bound slot
    ctx.setCalibSlots([3], [cams[1].K], cams=[1]); ctx.setCalibSlots([3], [cams[1].K], cams=[3])  # a slot without reference or map may change size
    with pytest.raises(api.SdvError, match="error -1"):
        ctx.setCalibSlots([0, 1], [cams[1].K, cams[1].K], cams=[1, 8])                          # camera out of range: all-or-nothing
    assert L.sdv_set_calib_slots_cams(ctx.p, 1, np.array([1], np.int32), None, np.array([1], np.int32).ctypes.data) == ERR_ARG   # no K on camera 1
    ctx.close()
    # frame / slot size mismatches in the mixed context of the fixture (slots 0-2: 1400x360, 3-5: 1200x360, 6-8: 1244x356)
    c0, c1 = cams[0], cams[1]
    clouds = [api.CoarseTracker(mixed, 0).cloud(l) for l in range(LEVELS)]
    with pytest.raises(api.SdvError, match="error -1"):
        api.CoarseTracker(mixed, 0).setCoarseTrackingRef(c1.ids[3], c1.p4, c1.rh)
    assert all(all(_same(x, y) for x, y in zip(a, api.CoarseTracker(mixed, 0).cloud(l))) for l, a in enumerate(clouds))
    T = _track_inits(c0, 1)[0]; tr = api.CoarseTracker(mixed, 0)
    r0 = tr.calcRes(c0.ids[4], 1, T, 0.0, 0.0, 20.0); H0 = tr.calcGSSSE(1)
    with pytest.raises(api.SdvError, match="error -1"):
        tr.calcRes(c1.ids[4], 1, T, 0.0, 0.0, 20.0)
    assert _same(tr.calcGSSSE(1)[0], H0[0]) and _same(tr.calcGSSSE(1)[1], H0[1])
    Tb = np.stack([T, T]); ab = np.zeros((2, 2)); Tb0 = Tb.copy()
    for slots, frames in (([0, 3], [c0.ids[4], c0.ids[4]]), ([3, 0], [c1.ids[4], c1.ids[4]])):
        with pytest.raises(api.SdvError, match="error -1"):
            mixed.trackBatch(slots, frames, Tb, ab)
        assert _same(Tb, Tb0) and not ab.any()
    with pytest.raises(api.SdvError, match="error -1"):
        tr.trackNewestCoarse(c1.ids[4], T, [0.0, 0.0])
    job = dict(frame=c1.ids[6], sprelast_c2w=c1.poses[4], slast_c2w=c1.poses[5], lastF_c2w=c1.poses[3], aff_last=[0.0, 0.0], poses_valid=1, lastCoarseRMSE=[100.0] * 5)
    with pytest.raises(api.SdvError, match="error -1"):
        api.trackNewCoarseBatch(mixed, [dict(job, slot=3), dict(job, slot=1)])
    before = mrp.reprojectMap(0, c0.ids[7], c0.poses[7])
    with pytest.raises(api.SdvError, match="error -1"):
        mrp.setMap(0, [c0.ids[0], c1.ids[1]], c0.hT[:2], c0.hab[:2], c0.pts[c0.pts["host"] < 2])
    after = mrp.reprojectMap(0, c0.ids[7], c0.poses[7])
    assert _same(before[0], after[0]) and _same(before[1], after[1])
    with pytest.raises(api.SdvError, match="error -1"):
        mrp.reprojectMapBatch([0, 3], [c0.ids[7], c0.ids[7]], np.stack([c0.poses[7]] * 2))
    with pytest.raises(api.SdvError, match="error -1"):
        mrp.refineBatch([6, 0], [c1.ids[7], c0.ids[7]], np.stack([c1.poses[7], c0.poses[7]]))
    # a BA window of mixed sizes; the window in place stays as it was
    win = synth.make_ba_window(c0.seq, [0, 1, 2], n_per_frame=60, seed=1)
    gb = api.EnergyFunctional(mixed, win, c0.ids[:3], window=3); fr = gb.frames()
    with pytest.raises(api.SdvError, match="error -1"):
        api.EnergyFunctional(mixed, win, [c0.ids[0], c1.ids[1], c0.ids[2]], window=3)
    assert _same(gb.frames()["T_eval"], fr["T_eval"])
    # keyframe-rate stages work at the context size only
    with pytest.raises(api.SdvError, match="error -1"):
        api.immatureInit(mixed, c1.ids[0], [[100, 100], [200, 150]])
    assert len(api.immatureInit(mixed, c0.ids[0], [[100, 100], [200, 150]])) == 2
    pts = api.immatureInit(mixed, c0.ids[0], [[100, 100]])
    with pytest.raises(api.SdvError, match="error -1"):
        api.traceOnBatch(mixed, [c1.ids[1]], [0, 1], np.eye(3, dtype=np.float32), np.zeros(3, np.float32), np.array([1.0, 0.0], np.float32), pts)


# ------------------------------------------------------------------------------------------------ end to end
def test_end_to_end_raw_kitti360_and_kitti_in_one_batch():
    """raw KITTI-360 and KITTI drives, one mixed raw batch per step, trackNewCoarseBatch with the refinement: the poses of two per-size contexts, bit for bit"""
    api, synth = _mods()
    unds = [_mirror(CALIBS["kitti360"]), _mirror(CALIBS["kitti00"])]
    NF, S = 5, 2                                                                      # frames per drive (0 = keyframe), sequences per camera
    drives = []
    for c, u in enumerate(unds):
        seed = 3100 + 37 * c
        K_raw = tuple(float(v) for v in CALIBS["kitti360" if c == 0 else "kitti00"].split()[1:5]); rs = cached_sequence(NF, seed, K_raw, (u.wOrg, u.hOrg))
        raw = [np.ascontiguousarray(im.astype(np.uint8)) for im in rs.images]
        rect0 = u.undistort_host(raw[0])
        cloud = synth.lidar_pixels(synth.World(seed), rs.R[0], rs.t[0], u.K4, (u.w, u.h))
        pts = synth.select_points(rect0, cloud, 2000)
        p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
        mp = np.zeros(len(pts), api.MAP_PT_DTYPE); mp["u"], mp["v"], mp["idepth"] = pts[:, 0], pts[:, 1], pts[:, 2]
        drives.append(dict(raw=raw, p4=p4, rh=np.zeros(len(p4), np.int32), map=mp))
    I7 = np.array([1.0, 0, 0, 0, 0, 0, 0])

    def run(ctx, seqs, order):
        """seqs: (slot, camera) of each sequence; one ingest + one trackNewCoarseBatch per step; returns (camToWorld, n_matches, tries) per step and sequence"""
        rp = api.Reprojector(ctx); cams = sorted({c for _, c in seqs})
        fid = lambda c, k: 1000 * (c + 1) + k
        ctx.makeImagesBatch([fid(c, 0) for c in cams], [drives[c]["raw"][0].ctypes.data for c in cams], raw=True, cams=cams)
        for s, c in seqs:
            api.CoarseTracker(ctx, s).setCoarseTrackingRef(fid(c, 0), drives[c]["p4"], drives[c]["rh"])
            rp.setMap(s, [fid(c, 0)], I7[None], None, drives[c]["map"])
        hist = {s: [I7, I7] for s, _ in seqs}; out = []
        for k in range(1, NF):
            ctx.makeImagesBatch([fid(c, k) for c in cams], [drives[c]["raw"][k].ctypes.data for c in cams], raw=True, cams=cams)
            jobs = [dict(slot=s, frame=fid(c, k), sprelast_c2w=hist[s][-2], slast_c2w=hist[s][-1], lastF_c2w=I7, aff_last=[0.0, 0.0],
                         poses_valid=0 if k == 1 else 1, lastCoarseRMSE=[100.0] * 5) for s, c in seqs]
            r = api.trackNewCoarseBatch(ctx, jobs, cell_order=order)
            for (s, _), o in zip(seqs, r):
                hist[s].append(o["camToWorld"])
            out.append([(o["camToWorld"], o["n_matches"], o["tries"]) for o in r])
        return out

    mixed = api.Context(unds[0].K4, unds[0].w, unds[0].h, n_tracker_slots=2 * S, max_frames=4 * NF, max_kf_images=8)
    mixed.setCameraSize(1, unds[1].w, unds[1].h)
    for c, u in enumerate(unds):
        mixed.setUndistort(u, cam=c)
    mixed.setCalibSlots(list(range(S, 2 * S)), [unds[1].K4] * S, cams=[1] * S)
    order = np.random.default_rng(8).permutation(api.Reprojector(mixed).n_cells).astype(np.int32)
    seqs = [(0, 0), (S, 1), (1, 0), (S + 1, 1)]                                       # cameras interleaved in every batch
    got = run(mixed, seqs, order)
    for c, u in enumerate(unds):
        one = api.Context(u.K4, u.w, u.h, n_tracker_slots=S, max_frames=2 * NF, max_kf_images=8)
        one.setUndistort(u, cam=c)                                                    # camera c of a context of its own size: the same handles and tables
        want = run(one, [(j, c) for j in range(S)], filtered_order(order, c))
        for k in range(NF - 1):
            mine = [g for (_, cc), g in zip(seqs, got[k]) if cc == c]
            for a, b in zip(mine, want[k]):
                assert _same(a[0], b[0]) and a[1:] == b[1:] and b[1] > 10, (c, k, a[1:], b[1:])
        one.close()
    mixed.close()
