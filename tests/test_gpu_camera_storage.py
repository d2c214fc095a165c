"""GPU tests (-m gpu) of frame storage per camera (sdv_set_camera_storage, sdv_camera_storage_bytes).

The context is INTEGRATION.md's three-dataset one: 1400x1024 at 5 levels.  Camera 1 is KITTI 00 (1200x360, raw tables of calib/KITTI/00.txt).  The same mixed
workload runs in a context where camera 1 has a pool of its own and in one where it has none; every result must be bit-identical.  The rules of the pools
(capacity without fallback, moving handles, refusals that change nothing) and the byte counts the library reports are checked on their own."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from test_undistort import CALIBS, _check_levels, _mirror
from test_gpu_mixed_sizes import Cam, _track_inits

pytestmark = pytest.mark.gpu

CTX = (1400, 1024)
LEVELS = 5
KITTI = (1200, 360)
FORMATS = ["host_f32", "host_u8", "dev_f32", "dev_u8", "adopt"]
MIX = [1, 0, 1, 1, 0, 1]                                   # camera of each image of a mixed ingest batch
ERR_ARG, ERR_STATE = -1, -5
CTX_BYTES = (15253760, 22937600)                           # one frame / one keyframe level-0 image at 1400x1024, 5 levels


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _context(api, synth, pool, n_slots=4, max_frames=64, max_kf_images=64, cam_frames=48, cam_kf=48):   # read-back builds level-0 texels: room for every frame
    ctx = api.Context(synth.K360_K, *CTX, levels=LEVELS, n_tracker_slots=n_slots, max_frames=max_frames, max_kf_images=max_kf_images)
    ctx.setCameraSize(1, *KITTI)
    if pool:
        ctx.setCameraStorage(1, cam_frames, cam_kf)
    return ctx


def _images(mix, seed):
    rng = np.random.default_rng(seed); out = []
    for k, c in enumerate(mix):
        w, h = CTX if c == 0 else KITTI
        if k % 2:
            out.append(rng.integers(0, 256, (h, w)).astype(np.uint8))
        else:
            yy, xx = np.mgrid[0:h, 0:w]; out.append(((xx * 3 + yy * 5 + 7 * k) % 256).astype(np.uint8))
    return out


def _ingest(ctx, ids, imgs8, fmt, cams, keep):
    import torch
    f32 = [np.ascontiguousarray(i.astype(np.float32)) for i in imgs8]
    if fmt == "host_f32":
        ctx.makeImagesBatch(ids, [a.ctypes.data for a in f32], cams=cams)
    elif fmt == "host_u8":
        ctx.makeImagesBatch(ids, [a.ctypes.data for a in imgs8], u8=True, cams=cams)
    else:
        ts = [torch.from_numpy(a if fmt == "dev_u8" else b).cuda() for a, b in zip(imgs8, f32)]; torch.cuda.synchronize(); keep.extend(ts)
        ctx.makeImagesBatch(ids, [t.data_ptr() for t in ts], device=True, u8=fmt == "dev_u8", adopt=fmt == "adopt", cams=cams)
    ctx.sync()
    return f32


def _levels(ctx, fid):
    return [ctx.frameLevel(fid, l) for l in range(ctx.camLevels(ctx.frame_cam.get(fid, 0)))]


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


# ------------------------------------------------------------------------------------------------ bit-identity
def _ingest_workload(api, ctx, check_oracle):
    """mixed batches of every format, a raw batch and a re-ingest that changes cameras; every level of every frame"""
    und = _mirror(CALIBS["kitti00"]); ctx.setUndistort(und, cam=1)
    keep, got, fid = [], {}, 0
    for i, fmt in enumerate(FORMATS):
        imgs8 = _images(MIX, 40 + i); ids = list(range(fid, fid + len(MIX))); fid += len(MIX)
        want = _ingest(ctx, ids, imgs8, fmt, MIX, keep)
        for k, f in enumerate(ids):
            if check_oracle and MIX[k] == 1:
                _check_levels(api, ctx, f, want[k], LEVELS)
            got[(fmt, f)] = _levels(ctx, f)
    rng = np.random.default_rng(6); raws = [rng.integers(0, 256, (und.hOrg, und.wOrg)).astype(np.uint8) for _ in range(3)]
    ids = list(range(fid, fid + 3)); fid += 3
    ctx.makeImagesBatch(ids, [r.ctypes.data for r in raws], raw=True, cams=[1, 1, 1]); ctx.sync()
    for k, f in enumerate(ids):
        if check_oracle:
            _check_levels(api, ctx, f, und.undistort_host(raws[k]), LEVELS)
        got[("raw", f)] = _levels(ctx, f)
    mix2 = [1 - c for c in MIX]; imgs8 = _images(mix2, 99); ids = list(range(len(MIX)))                 # handles of the first batch change cameras (and pools)
    _ingest(ctx, ids, imgs8, "host_f32", mix2, keep)
    for f in ids:
        got[("moved", f)] = _levels(ctx, f)
    for f in range(fid):
        ctx.releaseFrame(f)
    return got


def test_ingest_every_format_bit_identical_with_and_without_pool():
    api, synth = _mods()
    a, b = _context(api, synth, False), _context(api, synth, True)
    ga = _ingest_workload(api, a, False); gb = _ingest_workload(api, b, True)
    assert ga.keys() == gb.keys()
    for key in ga:
        assert all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(ga[key], gb[key])), key
    a.close(); b.close()


def _track_workload(api, synth, ctx):
    """camera-1 sequences on slots 0..2: trackBatch, trackNewCoarseBatch, refineBatch"""
    cam = Cam(api, synth, 1, tuple(synth.KITTI_K)); out = {}
    ctx.setCalibSlots([0, 1, 2], [cam.K] * 3, cams=[1] * 3)
    rp = cam.load(api, ctx, [0, 1, 2], 1)
    T = _track_inits(cam, 3); ab = np.zeros((3, 2)); ab[1] = [0.02, 1.0]
    r = ctx.trackBatch([0, 1, 2], [cam.ids[4]] * 3, T, ab)
    out["track"] = (T, ab, r["good"], r["flow"], r["iterations"], r["accepts"], r["evals"], r["lastResiduals"])
    order = np.random.default_rng(4).permutation(rp.n_cells).astype(np.int32); P = cam.poses
    base = dict(frame=cam.ids[6], sprelast_c2w=P[4], slast_c2w=P[5], lastF_c2w=P[3], aff_last=[0.0, 0.0])
    jobs = [dict(base, slot=0, poses_valid=1, lastCoarseRMSE=[100.0] * 5), dict(base, slot=1, poses_valid=1, lastCoarseRMSE=[1e-3] * 5),
            dict(base, slot=2, poses_valid=0, lastCoarseRMSE=[100.0] * 5, frame=cam.ids[4])]
    out["new_coarse"] = [[g[k] for k in sorted(g)] for g in api.trackNewCoarseBatch(ctx, jobs, cell_order=order)]
    rng = np.random.default_rng(3); T0 = np.stack([P[7] + np.concatenate([np.zeros(4), rng.normal(0, 0.04, 3)]) for _ in range(3)])
    f = rp.refineBatch([0, 1, 2], [cam.ids[7]] * 3, T0, cell_order=order, max_matches=150)
    out["refine"] = [f[k] for k in ("T", "n_matches", "res", "iterations", "accepts")]
    assert r["good"].all() and (f["n_matches"] > 10).all()
    return out


def _ba_workload(api, synth, ctx):
    """a camera-1 window: optimize_batch, then the keyframe hand-over"""
    seq = cached_sequence(8, 2001, tuple(synth.KITTI_K), KITTI); kfs = [0, 1, 2, 3, 4, 5, 6]
    win = synth.make_ba_window(seq, kfs, n_per_frame=180, seed=21, pose_noise=(0.005, 0.0003), match_noise=0.2, prior_scale=1e-3)
    ids = [500 + k for k in kfs]
    for k, f in zip(kfs, ids):
        ctx.makeImages(f, seq.images[k], cam=1)
    gb = api.EnergyFunctional(ctx, win, ids, window=0); r = api.optimize_batch(ctx, [0], 6); fr = gb.frames()
    out = dict(opt=(r["iterations"], r["accepts"], r["rmse"], fr["T_eval"], fr["state"], gb.points()["idepth"]))
    sel = (win["host"] == 1).astype(np.int32); sel[::4] = 1; sel[win["host"] == win["nF"] - 1] = 0
    out["flag"] = gb.flagPointsForRemoval(sel); m = gb.marginalizePointsF(); out["marg"] = [m[k] for k in ("M", "Mb", "Msc", "Mbsc")]
    gb.marginalizeFrame(1); out["prior"] = list(gb.prior())
    assert r["accepts"][0] > 0
    return out


def _keyframe_workload(api, synth, ctx):
    """a camera-1 keyframe step: LiDAR handler, makeNewTraces, traceOn into the next frames, activation"""
    K = tuple(synth.KITTI_K); seq = cached_sequence(4, 5101, K, KITTI)
    ims = [np.ascontiguousarray(im, np.float32) for im in seq.images]; ids = [700 + k for k in range(4)]
    ctx.makeImagesBatch(ids, [a.ctypes.data for a in ims], cams=[1] * 4); ctx.sync()
    poses = [np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(4)]
    w_, R, t = synth.World(5200), *synth.trajectory(2, 5200); S = [synth.lidar_sweep(w_, R[0], t[0], seed=10)]
    lid = api.LidarFrontEnd(ctx).handle(S, synth.RLC, synth.TLC, np.array([K], np.float32), [[10000, -1, 10000, -1]], cams=[1])
    ps = api.PixelSelector(ctx, 1, api.random_pattern(*CTX), cams=[1])
    dl = [api.lidar_density(lid[0]["lrud"], KITTI, 1500.0)]
    res, num = ps.makeNewTracesBatch([0], [ids[0]], [lid[0]["cloud_px"]], dl, 1500.0, [lid[0]["addFeaturePoint"]], cap=1 << 15)
    pts = res[0][1].copy(); pb = np.array([0, len(pts)], np.int32); sts = []
    for k in (1, 2):
        g = orc.trace_geometry(K, poses[0], poses[k])
        sts.append(api.traceOnBatch(ctx, [ids[k]], pb, g[0][None], g[1][None], g[2][None], pts, cams=[1]))
    good = pts["lastTraceStatus"] == api.IPS_GOOD
    K0, K1 = orc.distmap_geometry(K, None, None); Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
    Rr, tr = synth.rel_pose(seq.R[0], seq.t[0], seq.R[3], seq.t[3]); A = (K1 @ Rr.astype(np.float32) @ Ki0).astype(np.float32); B = (K1 @ tr.astype(np.float32)).astype(np.float32)
    cl = lid[0]["cloud_px"][::5]; uvid = np.stack([np.floor(cl[:, 0]), np.floor(cl[:, 1]), 1.0 / cl[:, 2]], 1).astype(np.float32)
    cand4 = np.stack([pts["u"][good], pts["v"][good], 0.5 * (pts["idepth_max"][good] + pts["idepth_min"][good]), res[0][0]["my_type"][good]], 1).astype(np.float32)
    decs, maps = api.activateSelectBatch(ctx, [dict(pt_begin=[0, len(uvid)], KRKi=A[None], Kt=B[None], uvid=uvid, cand_begin=[0, len(cand4)], cKRKi=A[None], cKt=B[None],
                                                    cand4=cand4, minActDist=2.0)], want_maps=True, cams=[1])
    assert len(pts) > 100 and 1 in decs[0].tolist()
    return dict(lid=(lid[0]["cloud_px"], lid[0]["lrud"]), rec=res[0][0].tobytes(), num=num[0], pts=pts.tobytes(), st=sts, map=ps.selectionMap(0), dec=decs[0], dmap=maps[0])


def _flatten(x):
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _flatten(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for e in x for v in _flatten(e)]
    return [x]


@pytest.mark.parametrize("stage", ["track", "ba", "keyframe"])
def test_camera1_stages_bit_identical_with_and_without_pool(stage):
    api, synth = _mods(); run = dict(track=_track_workload, ba=_ba_workload, keyframe=_keyframe_workload)[stage]
    outs = []
    for pool in (False, True):
        ctx = _context(api, synth, pool)
        a = ctx.cameraStorageBytes(1)
        outs.append(_flatten(run(api, synth, ctx)))
        assert a == ((4596000, 6912000) if pool else CTX_BYTES)
        ctx.close()
    assert len(outs[0]) == len(outs[1])
    for k, (x, y) in enumerate(zip(*outs)):
        assert (x == y) if isinstance(x, (bytes, int, float, str)) else _same(x, y), (stage, k)


# ------------------------------------------------------------------------------------------------ bytes
def test_storage_bytes_match_the_allocation_sizes():
    api, synth = _mods()
    ctx = api.Context(synth.K360_K, *CTX, levels=LEVELS, max_frames=4, max_kf_images=2)
    for c, wh in ((1, KITTI), (2, (1400, 360)), (3, (1392, 1024))):
        ctx.setCameraSize(c, *wh)
    for c in range(4):
        assert ctx.cameraStorageBytes(c) == CTX_BYTES, c
    for c in (1, 2, 3):
        ctx.setCameraStorage(c, 2, 1)
    assert ctx.cameraStorageBytes(0) == CTX_BYTES
    assert ctx.cameraStorageBytes(1) == (4596000, 6912000)
    assert ctx.cameraStorageBytes(2) == (5361780, 8064000)
    assert ctx.cameraStorageBytes(3) == (15167232, 22806528)
    ctx.setCameraStorage(1, 0, 0)
    assert ctx.cameraStorageBytes(1) == CTX_BYTES
    ctx.close()


# ------------------------------------------------------------------------------------------------ rules
def _img(c, seed):
    w, h = CTX if c == 0 else KITTI
    return np.random.default_rng(seed).uniform(0, 255, (h, w)).astype(np.float32)


def test_capacity_has_no_fallback():
    api, synth = _mods(); L = api.LIB
    ctx = _context(api, synth, True, max_frames=3, max_kf_images=3, cam_frames=3, cam_kf=2)
    for f in range(3):
        ctx.makeImages(10 + f, _img(1, f), cam=1)
    with pytest.raises(api.SdvError, match="error -4.*camera 1"):
        ctx.makeImages(13, _img(1, 3), cam=1)
    for f in range(3):                                                                         # no context frame was taken
        ctx.makeImages(20 + f, _img(0, f))
    with pytest.raises(api.SdvError, match="error -4"):
        ctx.makeImages(23, _img(0, 3))
    # keyframe images: a window of three camera-1 frames needs three of the pool's two
    seq = cached_sequence(3, 2002, tuple(synth.KITTI_K), KITTI); win = synth.make_ba_window(seq, [0, 1, 2], n_per_frame=60, seed=1)
    for k in range(3):
        ctx.makeImages(10 + k, seq.images[k], cam=1)
    with pytest.raises(api.SdvError, match="error -4.*camera 1"):
        api.EnergyFunctional(ctx, win, [10, 11, 12])
    for f in (11, 12):
        ctx.releaseFrame(f)
    assert L.sdv_set_camera_storage(ctx.p, 1, 4, 4) == ERR_STATE                                 # frame 10 resident (and its keyframe image taken)
    ctx.releaseFrame(10)
    ctx.setCameraStorage(1, 4, 4)
    for k in range(3):
        ctx.makeImages(10 + k, seq.images[k], cam=1)
    api.EnergyFunctional(ctx, win, [10, 11, 12])                                                 # the new pool has room for the window
    ctx.close()


def test_handles_move_between_pools():
    api, synth = _mods(); L = api.LIB
    ctx = _context(api, synth, True, max_frames=2, max_kf_images=2, cam_frames=2, cam_kf=2)
    ctx.makeImages(1, _img(0, 1)); ctx.makeImages(2, _img(0, 2))
    ref = api.Context(synth.KITTI_K, *KITTI, levels=LEVELS, max_frames=2, max_kf_images=2)
    ref.makeImages(1, _img(1, 5))
    ctx.makeImages(1, _img(1, 5), cam=1)                                                         # handle 1 moves into camera 1's pool ...
    ctx.makeImages(3, _img(0, 3))                                                                # ... and its context frame is free again
    assert all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(_levels(ctx, 1), _levels(ref, 1)))
    ctx.makeImages(4, _img(1, 4), cam=1)
    with pytest.raises(api.SdvError, match="error -4"):                                         # camera 1's pool is full: handle 2 stays where it was
        ctx.makeImages(2, _img(1, 6), cam=1)
    assert ctx.frame_cam.get(2, 0) == 0 and _same(ctx.frameLevel(2, 0)[0][..., 0], _img(0, 2))
    with pytest.raises(api.SdvError, match="error -4"):                                         # context pool full (2 and 3): handle 1 stays in camera 1's pool
        ctx.makeImages(1, _img(0, 7))
    assert _same(ctx.frameLevel(1, 0)[0][..., 0], _img(1, 5))
    # a pinned handle cannot move
    seq = cached_sequence(3, 2002, tuple(synth.KITTI_K), KITTI); win = synth.make_ba_window(seq, [0, 1], n_per_frame=60, seed=1)
    ctx.makeImages(1, seq.images[0], cam=1); ctx.makeImages(4, seq.images[1], cam=1)
    gb = api.EnergyFunctional(ctx, win, [1, 4]); before = ctx.frameLevel(1, 0)
    ctx.releaseFrame(3)
    arr = np.ascontiguousarray(_img(0, 8)); ids = np.array([1], np.uint64)
    assert L.sdv_frame_upload_batch(ctx.p, 1, ids, (api._vp * 1)(arr.ctypes.data), np.ones(1, np.float32)) == ERR_STATE
    assert all(_same(x, y) for x, y in zip(before, ctx.frameLevel(1, 0))) and gb.frames() is not None
    ref.close(); ctx.close()


def test_refused_batch_moves_no_handle():
    """a batch that moves handle 1 into camera 1's pool and then overflows that pool is refused as a whole: handle 1 keeps its context frame and image"""
    api, synth = _mods()
    ctx = _context(api, synth, True, max_frames=2, max_kf_images=2, cam_frames=1, cam_kf=1)
    ctx.makeImages(1, _img(0, 1)); before = _levels(ctx, 1)
    a, b = np.ascontiguousarray(_img(1, 2)), np.ascontiguousarray(_img(1, 3))
    with pytest.raises(api.SdvError, match="error -4.*camera 1"):
        ctx.makeImagesBatch([1, 2], [a.ctypes.data, b.ctypes.data], cams=[1, 1])
    assert ctx.frame_cam.get(1, 0) == 0 and all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(before, _levels(ctx, 1)))
    with pytest.raises(api.SdvError, match="error -3"):                                         # handle 2 was never claimed
        ctx.frameLevel(2, 0)
    ctx.makeImages(3, _img(0, 4))                                                                # the context pool's second frame is still free
    ctx.makeImagesBatch([1], [a.ctypes.data], cams=[1]); ctx.sync()                              # alone, the move fits
    ctx.makeImages(4, _img(0, 5))                                                                # and frees handle 1's context frame
    ctx.close()


def test_refusals_change_nothing():
    api, synth = _mods(); L = api.LIB
    ctx = _context(api, synth, True, max_frames=2, max_kf_images=2, cam_frames=2, cam_kf=1)
    ctx.makeImages(1, _img(1, 1), cam=1); lv = _levels(ctx, 1); b1 = ctx.cameraStorageBytes(1)
    for cam, n, k in ((0, 2, 1), (8, 2, 1), (-1, 2, 1), (2, -1, 0), (2, 2, -1)):
        assert L.sdv_set_camera_storage(ctx.p, cam, n, k) == ERR_ARG, (cam, n, k)
    for n in (0, 3):
        assert L.sdv_set_camera_storage(ctx.p, 1, n, 0) == ERR_STATE, n                           # replacing or dropping under a resident frame
    assert L.sdv_set_camera_size(ctx.p, 1, 1000, 300) == ERR_STATE                               # the pool has the camera's current size
    for c in range(8):
        if c != 1:
            assert ctx.cameraStorageBytes(c) == CTX_BYTES, c
    assert L.sdv_camera_storage_bytes(ctx.p, 8, None, None) == ERR_ARG
    assert ctx.cameraStorageBytes(1) == b1 == (4596000, 6912000)
    assert all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(lv, _levels(ctx, 1)))
    ctx.makeImages(2, _img(1, 2), cam=1)                                                         # the pool still holds two frames
    with pytest.raises(api.SdvError, match="error -4"):
        ctx.makeImages(3, _img(1, 3), cam=1)
    ctx.makeImages(3, _img(0, 3)); ctx.makeImages(4, _img(0, 4))                                 # and the context pool its two
    # dropped: camera 1's frames come from the context pool again
    for f in (1, 2, 3, 4):
        ctx.releaseFrame(f)
    assert L.sdv_set_camera_size(ctx.p, 1, 1000, 300) == ERR_STATE                               # no resident frame: the pool alone refuses it
    assert ctx.cameraStorageBytes(1) == b1
    ctx.setCameraStorage(1, 0, 0); ctx.setCameraSize(1, 1000, 300); ctx.setCameraSize(1, *KITTI)
    assert ctx.cameraStorageBytes(1) == CTX_BYTES
    ctx.makeImages(1, _img(1, 1), cam=1); ctx.makeImages(2, _img(0, 2))
    with pytest.raises(api.SdvError, match="error -4"):
        ctx.makeImages(3, _img(1, 3), cam=1)
    assert all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(lv, _levels(ctx, 1)))      # same levels from context storage
    ctx.close()
