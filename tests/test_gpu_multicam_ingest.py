"""GPU tests (-m gpu) of the RAW ingest for several cameras in one context (sdv_set_undistort_cam + sdv_frame_upload_batch_raw_u8_cams).

The KITTI odometry calibrations come in three raw sizes that all crop to 1200x360 with different rectified K (calib/KITTI/00.txt, 03.txt, 04.txt).
One context holds all three cameras plus a fourth with a response function and an inverse vignette; one raw batch interleaves them.  Every level of
every frame must equal, bit for bit, (a) the host mirror of Undistort::undistort<unsigned char> pushed through the oracle's makeImages and (b) the same
frame ingested by a fresh context that holds only that camera through the single-camera entries.  End to end, each sequence tracked in the mixed
context must give exactly what a per-camera context fed with host-rectified float frames gives."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from test_undistort import CALIBS, _check_levels, _mirror

pytestmark = pytest.mark.gpu

KITTI = [CALIBS["kitti00"], CALIBS["kitti03"],
         "Pinhole 707.0912 707.0912 601.8873 183.1104 0\n1226 370\ncrop\n1200 360\n"]    # calib/KITTI/04.txt of the reference, verbatim (4-line data file)
MIX = [0, 1, 2, 1, 0, 2, 3, 1, 3, 2, 0, 3, 1, 2]                                     # camera of each frame of the mixed batch
EXPOSURE = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.02, 1.0, 0.0, 1.0, 1.0, 0.5, 1.0, 1.0]    # camera 3: photometric branch (> 0) and factor branch (== 0)
N_CONTIG = 7                                                                       # frames 0..6 lie back to back in one host buffer (one coalesced copy of mixed sizes)


def _api():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api
    return api


def _cameras():
    """cameras 0-2: KITTI 00, 03, 04; camera 3: the 04 geometry with a response G and an inverse vignette (PhotometricUndistorter::processFrame :193-203)"""
    cams = [_mirror(t) for t in KITTI]
    u = _mirror(KITTI[2]); rng = np.random.default_rng(17)
    u.G = (255.0 * (np.arange(256) / 255.0) ** 1.6).astype(np.float32); u.vignetteMapInv = rng.uniform(0.8, 1.5, (u.hOrg, u.wOrg)).astype(np.float32)
    return cams + [u]


def _remap(u, src):
    """Undistort::undistort's bilinear remap of a float source image, in the reference's operation order (tests/test_undistort.py)"""
    xx = u.remapX.reshape(-1); yy = u.remapY.reshape(-1); ok = xx >= 0
    xs = np.where(ok, xx, np.float32(1)); ys = np.where(ok, yy, np.float32(1)); xi = xs.astype(np.int32); yi = ys.astype(np.int32); s = src.reshape(-1)
    fx = xs - xi.astype(np.float32); fy = ys - yi.astype(np.float32); xy = fx * fy; o = xi + yi * u.wOrg
    out = xy * s[o + 1 + u.wOrg] + (fy - xy) * s[o + u.wOrg] + (fx - xy) * s[o + 1] + (np.float32(1) - fx - fy + xy) * s[o]
    return np.where(ok, out, np.float32(0)).astype(np.float32).reshape(u.h, u.w)


def _want(u, raw, exposure, factor=1.0):
    if u.G is not None and exposure > 0:
        return _remap(u, (u.G[raw] * u.vignetteMapInv).astype(np.float32))
    return u.undistort_host(raw, factor)


def _raws(cams, mix, seed):
    """one raw image per entry of mix, native size of its camera: the first N_CONTIG back to back in one buffer, the others separate arrays"""
    rng = np.random.default_rng(seed); sizes = [cams[c].wOrg * cams[c].hOrg for c in mix]
    pool = np.empty(sum(sizes[:N_CONTIG]), np.uint8); out = []; off = 0
    for k, c in enumerate(mix):
        u = cams[c]
        img = rng.integers(0, 256, (u.hOrg, u.wOrg)).astype(np.uint8)
        if k % 3 == 2:
            yy, xx = np.mgrid[0:u.hOrg, 0:u.wOrg]; img = ((xx * 3 + yy * 5 + k) % 256).astype(np.uint8)    # smooth ramp: the interpolation weights matter everywhere
        if k < N_CONTIG:
            dst = pool[off:off + sizes[k]].reshape(u.hOrg, u.wOrg); dst[:] = img; img = dst; off += sizes[k]
        out.append(img)
    return pool, out


def _levels(ctx, fid, L):
    return [ctx.frameLevel(fid, l) for l in range(L)]


def _same_levels(a, b):
    return all(np.array_equal(x[0], y[0], equal_nan=True) and np.array_equal(x[1], y[1], equal_nan=True) for x, y in zip(a, b))


def _mixed_context(api, cams, levels=None, max_frames=64):
    u = cams[0]; ctx = api.Context(u.K4, u.w, u.h, levels=levels, max_frames=max_frames, max_kf_images=max_frames)   # frameLevel(., 0) holds a level-0 texel image per frame
    for c, uc in enumerate(cams):
        ctx.setUndistort(uc, cam=c)
    return ctx


def _single_camera_levels(api, u, raws, exposures, L, levels=None):
    """the frames ingested by a fresh context that holds only this camera, through the unchanged single-camera entries"""
    ctx = api.Context(u.K4, u.w, u.h, levels=levels, max_frames=len(raws) + 2, max_kf_images=len(raws) + 2); ctx.setUndistort(u)
    ctx.makeImagesBatch(list(range(len(raws))), [r.ctypes.data for r in raws], exposures=exposures, raw=True); ctx.sync()
    out = [_levels(ctx, i, L) for i in range(len(raws))]
    ctx.close()
    return out


def _check_batch(api, cams, levels):
    ctx = _mixed_context(api, cams, levels); L = ctx.levels
    pool, raws = _raws(cams, MIX, seed=23)
    ids = [100 + k for k in range(len(MIX))]
    ctx.makeImagesBatch(ids, [r.ctypes.data for r in raws], exposures=EXPOSURE, raw=True, cams=MIX); ctx.sync()
    got = {k: _levels(ctx, ids[k], L) for k in range(len(MIX))}
    for k, c in enumerate(MIX):
        _check_levels(api, ctx, ids[k], _want(cams[c], raws[k], EXPOSURE[k]), L)                              # (a) host mirror through the oracle's makeImages
    for c in range(len(cams)):
        ks = [k for k in range(len(MIX)) if MIX[k] == c]
        single = _single_camera_levels(api, cams[c], [raws[k] for k in ks], [EXPOSURE[k] for k in ks], L, levels)
        for k, s in zip(ks, single):
            assert _same_levels(got[k], s), (c, k)                                                             # (b) a context holding only that camera
    ctx.close()


def test_mixed_batch_every_level_bit_exact():
    _check_batch(_api(), _cameras(), None)


def test_mixed_batch_single_level_context():
    """levels == 1: the level-0 plane comes from pyr_remap0_kernel"""
    _check_batch(_api(), _cameras(), 1)


def test_consecutive_ingests_and_camera_replacement():
    """three mixed ingests back to back without a sync (both staging parities, staging growth, the next upload overlapping), then camera 1's tables
    replaced between two ingests: frames of the earlier ingest keep the old tables, frames of the later one get the new"""
    api = _api(); cams = _cameras(); ctx = _mixed_context(api, cams, max_frames=48); L = ctx.levels
    mixes = [[0, 2, 1], [1, 1, 0, 2, 3], [2, 0, 1, 3, 1, 0, 2, 1, 3]]                                        # growing total bytes
    keep = []; want = {}; fid = 0
    for i, mix in enumerate(mixes):
        pool, raws = _raws(cams, mix, seed=40 + i); ex = [0.0 if (k % 2 and c == 3) else 1.0 for k, c in enumerate(mix)]
        ids = list(range(fid, fid + len(mix))); fid += len(mix); keep.append((pool, raws))
        ctx.makeImagesBatch(ids, [r.ctypes.data for r in raws], exposures=ex, raw=True, cams=mix)
        for k, c in enumerate(mix):
            want[ids[k]] = _want(cams[c], raws[k], ex[k])
    # camera 1 -> the 04 geometry (another raw size) with factor 0.75, while the ingest above may still be running
    mix = [1, 0, 1, 2]; pool, raws = _raws(cams, mix, seed=50); ids_a = list(range(fid, fid + 4)); fid += 4; keep.append((pool, raws))
    ctx.makeImagesBatch(ids_a, [r.ctypes.data for r in raws], raw=True, cams=mix)
    new1 = _mirror(KITTI[2]); ctx.setUndistort(new1, factor=0.75, cam=1)
    for k, c in enumerate(mix):
        want[ids_a[k]] = _want(cams[c], raws[k], 1.0)
    cams_b = [cams[0], new1, cams[2], cams[3]]
    pool, raws = _raws(cams_b, mix, seed=51); ids_b = list(range(fid, fid + 4)); fid += 4; keep.append((pool, raws))
    ctx.makeImagesBatch(ids_b, [r.ctypes.data for r in raws], raw=True, cams=mix); ctx.sync()
    for k, c in enumerate(mix):
        want[ids_b[k]] = _want(cams_b[c], raws[k], 1.0, 0.75 if c == 1 else 1.0)
    for f, img in want.items():
        _check_levels(api, ctx, f, img, L)
    ctx.close()


def test_refusals_change_nothing():
    api = _api(); cams = _cameras(); u = cams[0]; L = api.pyr_levels(u.w, u.h)
    ctx = api.Context(u.K4, u.w, u.h, max_frames=8)
    for cam in (-1, 8):
        with pytest.raises(api.SdvError, match="error -1"):
            ctx.setUndistort(u, cam=cam)
        assert api.LIB.sdv_set_undistort_cam(ctx.p, cam, u.wOrg, u.hOrg, u.remapX.reshape(-1), u.remapY.reshape(-1), 1.0, None, None) == -1
    ctx.setUndistort(cams[0], cam=0); ctx.setUndistort(cams[1], cam=1)
    _, raws = _raws(cams, [0, 1], seed=60)
    ctx.makeImagesBatch([7], [raws[0].ctypes.data], raw=True, cams=[0]); ctx.sync()
    before = _levels(ctx, 7, L)
    _, other = _raws(cams, [1, 1], seed=61)
    for bad, err in (([1, -1], "error -1"), ([1, 8], "error -1"), ([1, 5], "error -5")):                     # camera 5 was never set: SDV_ERR_STATE
        with pytest.raises(api.SdvError, match=err):
            ctx.makeImagesBatch([7, 9], [other[0].ctypes.data, other[1].ctypes.data], raw=True, cams=bad)
        ctx.sync()
        assert _same_levels(_levels(ctx, 7, L), before), bad
        with pytest.raises(api.SdvError):
            ctx.frameLevel(9, 0)                                                                              # never claimed
    with pytest.raises(api.SdvError, match="error -5"):
        ctx.makeImagesBatch([9], [other[0].ctypes.data], raw=True, cams=[2])
    _check_levels(api, ctx, 7, cams[0].undistort_host(raws[0]), L)
    ctx.close()
    fresh = api.Context(u.K4, u.w, u.h, max_frames=4)
    with pytest.raises(api.SdvError, match="error -5"):                                                       # no camera at all: the single-camera entry as before
        fresh.makeImagesBatch([1], [raws[0].ctypes.data], raw=True)
    fresh.close()


def test_end_to_end_tracking_mixed_cameras():
    """a short raw drive per KITTI camera, all frames in ONE mixed raw batch, every sequence's slots bound to its camera's K, all slots in one trackBatch:
    bit-identical to per-camera contexts fed with host-rectified float frames"""
    api = _api()
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import synth
    cams = [_mirror(t) for t in KITTI]; u0 = cams[0]; w, h = u0.w, u0.h
    NF, S = 4, 3                                                                # frames per drive (0 = keyframe), slots per camera (tracking frames 1..3)
    drives = []
    for c, u in enumerate(cams):
        seed = 2100 + 37 * c
        K_raw = tuple(float(v) for v in KITTI[c].split()[1:5]); rs = cached_sequence(NF, seed, K_raw, (u.wOrg, u.hOrg))
        raw = [np.ascontiguousarray(im.astype(np.uint8)) for im in rs.images]
        rect = [u.undistort_host(r) for r in raw]
        cloud = synth.lidar_pixels(synth.World(seed), rs.R[0], rs.t[0], u.K4, (w, h))
        pts = synth.select_points(rect[0], cloud, 2000)
        p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
        rng = np.random.default_rng(seed); T = []
        for k in range(1, NF):                                                  # ground truth 0 -> k, perturbed like a constant-motion prediction error
            R, t = synth.rel_pose(rs.R[0], rs.t[0], rs.R[k], rs.t[k])
            T.append(synth.se3_mul7(synth.se3_exp7(np.concatenate([rng.normal(0, 0.02, 3), rng.normal(0, 0.001, 3)])), np.concatenate([synth._quat_from_R(R), t])))
        T = np.stack(T)
        drives.append(dict(raw=raw, rect=rect, p4=p4, rh=np.zeros(len(p4), np.int32), T=T, ab=np.zeros((S, 2))))

    mixed = api.Context(u0.K4, w, h, n_tracker_slots=S * len(cams), max_frames=NF * len(cams) + 2)
    ids, ptrs, mix = [], [], []
    for c, (u, d) in enumerate(zip(cams, drives)):
        mixed.setUndistort(u, cam=c)
        mixed.setCalibSlots([S * c + j for j in range(S)], [u.K4] * S)
    for k in range(NF):                                                          # frames interleaved over the cameras
        for c, d in enumerate(drives):
            ids.append(1000 * (c + 1) + k); ptrs.append(d["raw"][k].ctypes.data); mix.append(c)
    mixed.makeImagesBatch(ids, ptrs, raw=True, cams=mix)
    for c, d in enumerate(drives):
        for j in range(S):
            api.CoarseTracker(mixed, S * c + j).setCoarseTrackingRef(1000 * (c + 1), d["p4"], d["rh"])
    T = np.concatenate([d["T"] for d in drives]); ab = np.concatenate([d["ab"] for d in drives])
    rm = mixed.trackBatch(list(range(S * len(cams))), [1000 * (c + 1) + 1 + j for c in range(len(cams)) for j in range(S)], T, ab)
    for c, (u, d) in enumerate(zip(cams, drives)):
        f = api.Context(u.K4, w, h, n_tracker_slots=S, max_frames=NF + 2)
        for k in range(NF):
            f.makeImages(k, d["rect"][k])
        for j in range(S):
            api.CoarseTracker(f, j).setCoarseTrackingRef(0, d["p4"], d["rh"])
        Tf, abf = d["T"].copy(), d["ab"].copy()
        rf = f.trackBatch(list(range(S)), [1 + j for j in range(S)], Tf, abf)
        sl = slice(S * c, S * c + S)
        assert np.array_equal(T[sl], Tf) and np.array_equal(ab[sl], abf), c
        for key in ("good", "flow", "iterations", "accepts", "evals"):
            assert np.array_equal(rm[key][sl], rf[key]), (c, key)
        assert np.array_equal(rm["lastResiduals"][sl], rf["lastResiduals"], equal_nan=True), c
        assert (rf["evals"][:, 0] > 0).all(), c                                 # the comparison is between real tracking runs (level-0 point evaluations)
        f.close()
    mixed.close()
