"""GPU tests (-m gpu) of the batched tracker-reference build (sdv_tracker_set_ref_batch) and the batched map install (sdv_map_set_batch).

Every comparison is bit for bit: a batch must give each slot exactly the clouds, counts and tracking results that one sdv_tracker_set_ref /
sdv_map_set per slot gives in a twin context, and the oracle's / the reference's clouds where those are compared."""
import os
import numpy as np
import pytest
import orc
from conftest import SMALL_WH, cached_sequence

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tracker_small.npz")
ID7 = np.array([1, 0, 0, 0, 0, 0, 0.0])
HDI = np.array([1e-5, 1e-3, 1e30, np.inf, -1.0], np.float32)
CHUNK_BYTES = 512 << 20                 # the build's plane budget per chunk (DESIGN.md Round 13)


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def _rows(rng, w, h, n, hdi=None):
    u = rng.uniform(0, w - 1, n); v = rng.uniform(0, h - 1, n)                       # inside the image under both rounding rules
    idp = rng.uniform(0.01, 1.0, n); hd = np.exp(rng.uniform(np.log(1e-5), np.log(1e-1), n)) if hdi is None else np.full(n, hdi)
    return np.stack([u, v, idp, hd], 1).astype(np.float32), (rng.uniform(size=n) < 0.4).astype(np.int32)


def _hard_rows(rng, w, h, base):
    """bench-like rows plus the edge cases: one pixel hit 64 times with mixed rounding, splats in the 2 px border, every HdiF class, idepth <= 0 and NaN"""
    p, r = base
    hit = np.tile(np.array([[w / 2 + 0.3, h / 2 + 0.2, 0.5, 1e-3]], np.float32), (64, 1)); hit[:, 2] = rng.uniform(-0.2, 1.0, 64); hit[:, 3] = HDI[rng.integers(0, 5, 64)]
    hit_r = rng.integers(0, 2, 64).astype(np.int32)
    bu = np.concatenate([rng.uniform(0, 2, 40), rng.uniform(w - 2, w - 1e-3, 40), rng.uniform(0, w - 1e-3, 80)])
    bv = np.concatenate([rng.uniform(0, h - 1e-3, 80), rng.uniform(0, 2, 40), rng.uniform(h - 2, h - 1e-3, 40)])
    border = np.stack([bu, bv, rng.uniform(0.05, 1, 160), np.full(160, 1e-3)], 1).astype(np.float32)
    odd, odd_r = _rows(rng, w, h, 200); odd[:, 3] = HDI[rng.integers(0, 5, 200)]; odd[:50, 2] = -odd[:50, 2]; odd[50:60, 2] = 0; odd[60:80, 2] = np.nan
    P = np.concatenate([p, hit, border, odd]).astype(np.float32); R = np.concatenate([r, hit_r, np.zeros(160, np.int32), odd_r]).astype(np.int32)
    perm = rng.permutation(len(P)); return P[perm], R[perm]


class Rig:
    """two identical contexts (batch / singles) with cameras, slots bound to them and one reference frame per (camera, index)"""

    def __init__(self, api, wh, cams, slot_cams, n_frames=2, levels=None, **kw):
        self.api = api; self.ctxs = []; self.slot_cams = list(slot_cams); rng = np.random.default_rng(7)
        self.imgs = {}
        for cam, (cw, ch, cl) in cams.items():
            for k in range(n_frames):
                im = rng.uniform(0, 255, (ch, cw)).astype(np.float32); im[5, 7] = np.nan; self.imgs[(cam, k)] = im
        for _ in range(2):
            ctx = api.Context((700.0, 700.0, wh[0] / 2, wh[1] / 2), wh[0], wh[1], levels=levels, n_tracker_slots=len(slot_cams), max_frames=len(self.imgs) + 2, **kw)
            for cam, (cw, ch, cl) in cams.items():
                if cam:
                    ctx.setCameraSize(cam, cw, ch)
                ctx.setCameraLevels(cam, cl)
            n = len(slot_cams)
            ctx.setCalibSlots(list(range(n)), [(700.0, 700.0, cams[c][0] / 2, cams[c][1] / 2) for c in slot_cams], cams=slot_cams)
            for (cam, k), im in self.imgs.items():
                ctx.makeImages(self.fid(cam, k), im, cam=cam)
            self.ctxs.append(ctx)
        self.cams = cams

    @staticmethod
    def fid(cam, k):
        return 1000 * (cam + 1) + k

    def install(self, slots, frames, P, R, ab=None):
        """batch in context 0, one sdv_tracker_set_ref per slot in context 1; returns the batch's counts"""
        api = self.api; b, s = self.ctxs
        cnt = b.setCoarseTrackingRefBatch(slots, frames, P, R, ab)
        for j, sl in enumerate(slots):
            a = (0.0, 0.0) if ab is None else tuple(ab[j])
            api.CoarseTracker(s, sl).setCoarseTrackingRef(frames[j], P[j], R[j], *a)
        return cnt

    def same(self, slots, cnt=None):
        api = self.api; b, s = self.ctxs
        for j, sl in enumerate(slots):
            tb, ts = api.CoarseTracker(b, sl), api.CoarseTracker(s, sl)
            for l in range(tb.levels):
                cb, cs = np.stack(tb.cloud(l)), np.stack(ts.cloud(l))
                assert cb.tobytes() == cs.tobytes(), (j, sl, l, cb.shape, cs.shape)
                if cnt is not None:
                    assert cnt[j, l] == cb.shape[1]
            if cnt is not None:
                assert np.all(cnt[j, tb.levels:] == 0)

    def close(self):
        for c in self.ctxs:
            c.close()


def _kitti_rows(synth, seq, n=2000):
    p = synth.select_points(seq.images[0], seq.clouds[0], n)
    return np.concatenate([p, np.full((len(p), 1), 1e-3, np.float32)], 1).astype(np.float32), np.zeros(len(p), np.int32)


@pytest.mark.parametrize("kind", ["kitti_1400", "carla_levels", "hd_1920"])
def test_batch_equals_singles(kind, kitti_seq):
    """one batch of mixed cameras / depths equals its jobs one by one: clouds at every level and the true counts"""
    api, synth = _mods(); rng = np.random.default_rng(11)
    if kind == "kitti_1400":
        cams = {0: (1400, 360, 4), 1: (1200, 360, 4)}; wh = (1400, 360); levels = None
    elif kind == "carla_levels":
        cams = {0: (1392, 1024, 5), 1: (1392, 1024, 4)}; wh = (1392, 1024); levels = 5
    else:
        cams = {0: (1920, 1200, 5), 1: (1200, 360, 4)}; wh = (1920, 1200); levels = 5
    slot_cams = [0, 1, 1, 0, 1, 0, 1]
    rig = Rig(api, wh, cams, slot_cams, levels=levels)
    P, R, F = [], [], []
    for j, c in enumerate(slot_cams):
        cw, ch, _ = cams[c]
        if j == 0:
            base = _kitti_rows(synth, kitti_seq) if (cw, ch) == synth.KITTI_WH else _rows(rng, cw, ch, 2000)
            p, r = _hard_rows(rng, cw, ch, base)
        elif j == 1:
            p, r = _hard_rows(rng, cw, ch, _kitti_rows(synth, kitti_seq) if (cw, ch) == synth.KITTI_WH else _rows(rng, cw, ch, 1500))
        elif j == 2:
            p, r = np.zeros((0, 4), np.float32), np.zeros(0, np.int32)                       # empty job
        elif j == 3:
            p, r = _rows(rng, cw, ch, 1)                                                      # one splat
        elif j == 5 and kind == "hd_1920":
            p, r = _rows(rng, cw, ch, 32768)                                                  # a 32 768-splat 1920x1200 job
        else:
            p, r = _rows(rng, cw, ch, 700)
        P.append(p); R.append(r); F.append(rig.fid(c, 0))                                      # jobs of one camera share its reference frame
    ab = rng.uniform(-1, 1, (len(slot_cams), 2))
    slots = list(range(len(slot_cams)))[::-1]                                                 # slots in another order than their jobs
    Pj = [P[s] for s in slots]; Rj = [R[s] for s in slots]; Fj = [F[s] for s in slots]; abj = ab[slots]
    cnt = rig.install(slots, Fj, Pj, Rj, abj)
    rig.same(slots, cnt)
    assert cnt[slots.index(2)].sum() == 0 and cnt[slots.index(0), 0] > 1000
    # the reference frame, exposure and affine of every job: calcRes agrees bit for bit
    b, s = rig.ctxs
    for j, sl in enumerate(slots):
        c = slot_cams[sl]; f1 = rig.fid(c, 1)
        rb = api.CoarseTracker(b, sl).calcRes(f1, 0, ID7, 0.01, 0.5, 20.0); rs = api.CoarseTracker(s, sl).calcRes(f1, 0, ID7, 0.01, 0.5, 20.0)
        assert rb.tobytes() == rs.tobytes()
    rig.close()


def test_batch_against_oracle_and_golden(kitti_seq):
    """a subset against the oracle's setCoarseTrackingRef, and the golden reference clouds installed as one job of a batch"""
    api, synth = _mods(); rng = np.random.default_rng(3); w, h = synth.KITTI_WH; L = 4
    ctx = api.Context(synth.KITTI_K, w, h, n_tracker_slots=3, max_frames=3); ctx.makeImages(0, kitti_seq.images[0])
    p, r = _hard_rows(rng, w, h, _kitti_rows(synth, kitti_seq)); p2, r2 = _rows(rng, w, h, 900)
    ctx.setCoarseTrackingRefBatch([2, 0], [0, 0], [p, p2], [r, r2])
    f0 = orc.Frame(kitti_seq.images[0], L)
    for slot, (pp, rr) in ((2, (p, r)), (0, (p2, r2))):
        o = orc.CoarseTracker(w, h, L, synth.KITTI_K); o.setCoarseTrackingRef(f0, pp, rr)
        for l in range(L):
            assert np.stack(api.CoarseTracker(ctx, slot).cloud(l)).tobytes() == np.stack(o.cloud(l)).tobytes(), (slot, l)
    ctx.close()
    g = np.load(GOLD); w, h = SMALL_WH
    ctx = api.Context(tuple(g["K"]), w, h, n_tracker_slots=3, max_frames=3); ctx.makeImages(0, g["img0"].astype(np.float32)); ctx.makeImages(1, g["img1"].astype(np.float32))
    q1, s1 = _rows(rng, w, h, 500); q2, s2 = _rows(rng, w, h, 300)
    ctx.setCoarseTrackingRefBatch([1, 0, 2], [1, 0, 0], [q1, g["pts4"], q2], [s1, g["round_half"], s2], [[0, 0], list(g["ref_ab"]), [0, 0]])
    for l in range(4):
        assert np.array_equal(np.stack(api.CoarseTracker(ctx, 0).cloud(l)), g[f"cloud{l}"])
    ctx.close()


def _plane_bytes(w, h, L):
    return 8 * sum((w >> l) * (h >> l) for l in range(L))


def test_chunks_equal_singles():
    """a batch over at least three chunks of the plane budget, with a chunk boundary between jobs of different cameras"""
    api, _ = _mods(); rng = np.random.default_rng(21)
    cams = {0: (1400, 360, 4), 1: (1200, 360, 4)}
    per = {c: _plane_bytes(*cams[c]) for c in cams}
    n1 = CHUNK_BYTES // per[1]; n0 = CHUNK_BYTES // per[0]
    slot_cams = [1] * n1 + [0] * n0 + [1] * 30                          # chunk 1: n1 camera-1 jobs (the next, camera 0, does not fit); chunk 2: n0 camera-0 jobs
    rig = Rig(api, (1400, 360), cams, slot_cams, n_frames=1, max_ref_points=6000)
    P, R, F = [], [], []
    for c in slot_cams:
        p, r = _rows(rng, cams[c][0], cams[c][1], int(rng.integers(0, 400))); P.append(p); R.append(r); F.append(rig.fid(c, 0))
    slots = list(range(len(slot_cams)))
    cnt = rig.install(slots, F, P, R)
    rig.same(slots, cnt)
    rig.close()


def test_launch_count_fixed():
    """the launches of one call do not grow with the job count within a chunk, nor with colliding splats"""
    api, synth = _mods(); rng = np.random.default_rng(5); w, h = synth.KITTI_WH
    ctx = api.Context(synth.KITTI_K, w, h, n_tracker_slots=64, max_frames=2, max_ref_points=8192); ctx.makeImages(0, rng.uniform(0, 255, (h, w)).astype(np.float32))
    counts = []
    for n, collide in ((8, False), (64, False), (64, True), (8, True)):
        P, R = [], []
        for _ in range(n):
            p, r = _rows(rng, w, h, 1500)
            if collide:
                p[:500, :2] = p[0, :2]                                    # 500 splats on one pixel
            P.append(p); R.append(r)
        l0 = ctx.launch_count(); ctx.setCoarseTrackingRefBatch(list(range(n)), [0] * n, P, R); counts.append(ctx.launch_count() - l0)
    assert len(set(counts)) == 1 and counts[0] > 0, counts
    ctx.close()


def test_tracking_after_batched_install(kitti_seq):
    """trackBatch after a batched install gives the outputs of tracking after per-slot installs, bit for bit"""
    api, synth = _mods(); w, h = synth.KITTI_WH; rng = np.random.default_rng(9)
    outs = []
    for batched in (True, False):
        ctx = api.Context(synth.KITTI_K, w, h, n_tracker_slots=4, max_frames=4)
        for i in range(3):
            ctx.makeImages(i, kitti_seq.images[i])
        base = _kitti_rows(synth, kitti_seq); P = [base[0][k::2] for k in range(2)] * 2; R = [base[1][k::2] for k in range(2)] * 2
        ab = np.array([[0.0, 0.0], [0.01, 0.5], [0.0, 1.0], [-0.02, 0.0]])
        if batched:
            ctx.setCoarseTrackingRefBatch([0, 1, 2, 3], [0, 0, 1, 0], P, R, ab)
        else:
            for s, f in enumerate([0, 0, 1, 0]):
                api.CoarseTracker(ctx, s).setCoarseTrackingRef(f, P[s], R[s], *ab[s])
        T = np.tile(ID7, (4, 1)); a = np.zeros((4, 2))
        r = ctx.trackBatch([0, 1, 2, 3], [1, 2, 2, 2], T, a)
        outs.append((T, a, r)); ctx.close()
    (T0, a0, r0), (T1, a1, r1) = outs
    assert T0.tobytes() == T1.tobytes() and a0.tobytes() == a1.tobytes()
    for k in ("good", "lastResiduals", "flow", "evals", "iterations", "accepts"):
        assert np.asarray(r0[k]).tobytes() == np.asarray(r1[k]).tobytes(), k


def _raw_batch(api, ctx, slots, frames, pb, p4, rh, ab=None, npts=None):
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    return api.LIB.sdv_tracker_set_ref_batch(ctx.p, len(slots), i32(slots), np.ascontiguousarray(frames, np.uint64), i32(pb), np.ascontiguousarray(p4, np.float32),
                                             i32(rh), None if ab is None else np.ascontiguousarray(ab, np.float64).ctypes.data, npts)


def test_refusals_change_nothing():
    """every refusal returns its code before anything is enqueued: clouds and reference of every slot unchanged"""
    api, _ = _mods(); rng = np.random.default_rng(17)
    cams = {0: (1400, 360, 4), 1: (1200, 360, 4)}
    rig = Rig(api, (1400, 360), cams, [0, 1, 1], n_frames=2)
    ctx = rig.ctxs[0]; tr = [api.CoarseTracker(ctx, s) for s in range(3)]
    P = [_rows(rng, cams[c][0], cams[c][1], 800) for c in (0, 1, 1)]
    ctx.setCoarseTrackingRefBatch([0, 1, 2], [rig.fid(0, 0), rig.fid(1, 0), rig.fid(1, 0)], [p for p, _ in P], [r for _, r in P])

    def snap():
        return [[np.stack(t.cloud(l)).tobytes() for l in range(4)] + [t.calcRes(rig.fid(c, 1), 0, ID7, 0, 0, 20.0).tobytes()] for t, c in zip(tr, (0, 1, 1))]
    before = snap()
    p1, r1 = _rows(rng, 1200, 360, 100); p0, r0 = _rows(rng, 1400, 360, 100)
    pb = [0, 100, 200]; p4 = np.concatenate([p0, p1]); rh = np.concatenate([r0, r1])
    f0, f1 = rig.fid(0, 1), rig.fid(1, 1)
    out = np.zeros(2 * 6, np.int32)
    assert api.LIB.sdv_tracker_set_ref_batch(None, 2, np.array([0, 1], np.int32), np.array([f0, f1], np.uint64), np.array(pb, np.int32), p4, rh, None, out) == -1
    assert _raw_batch(api, ctx, [0, 1], [f0, f1], [5, 100, 200], p4, rh, npts=out) == -1          # pt_begin[0] != 0
    assert _raw_batch(api, ctx, [0, 1], [f0, f1], [0, 150, 100], p4, rh, npts=out) == -1          # decreasing
    assert _raw_batch(api, ctx, [0, 3], [f0, f1], pb, p4, rh, npts=out) == -1                     # slot out of range
    assert _raw_batch(api, ctx, [1, 1], [f1, f1], [0, 100, 200], np.concatenate([p1, p1]), np.concatenate([r1, r1]), npts=out) == -1   # slot twice
    assert _raw_batch(api, ctx, [0, 1], [f0, 77], pb, p4, rh, npts=out) == -3                     # unknown frame
    assert _raw_batch(api, ctx, [0, 1], [f0, f0], pb, p4, rh, npts=out) == -1                     # frame of another size than the slot's camera
    bad = p4.copy(); bad[150, 0] = 1300.0; bad[150, 1] = 10                                       # inside the 1400x360 context, outside camera 1's 1200x360
    assert _raw_batch(api, ctx, [0, 1], [f0, f1], pb, bad, rh, npts=out) == -1
    assert "job 1, row 50" in api.LIB.sdv_last_error(ctx.p).decode()
    assert snap() == before
    assert _raw_batch(api, ctx, [], [], [0], np.zeros(4), np.zeros(1), npts=np.zeros(1, np.int32)) == 0   # n == 0
    rig.close()


def test_over_capacity_installs_the_rest():
    """a job over max_ref_points is left without reference; every other job equals its single install"""
    api, _ = _mods(); rng = np.random.default_rng(19)
    cams = {0: (1200, 360, 4)}
    rig = Rig(api, (1200, 360), cams, [0, 0, 0], n_frames=2, max_ref_points=3000)
    P = [_rows(rng, 1200, 360, 400), _rows(rng, 1200, 360, 4000), _rows(rng, 1200, 360, 500)]
    b, s = rig.ctxs; fr = [rig.fid(0, 0)] * 3
    out = np.zeros(3 * 6, np.int32)
    rc = _raw_batch(api, b, [0, 1, 2], fr, [0, 400, 4400, 4900], np.concatenate([p for p, _ in P]), np.concatenate([r for _, r in P]), npts=out)
    assert rc == -4 and "job 1" in api.LIB.sdv_last_error(b.p).decode()
    assert out.reshape(3, 6)[1, 0] > 3000 and np.all(out.reshape(3, 6)[:, 4:] == 0)
    rs = np.zeros(6)
    assert api.LIB.sdv_tracker_calc_res(b.p, 1, rig.fid(0, 1), 0, ID7, 0, 0, 20.0, rs) == -5
    for sl in (0, 2):
        api.CoarseTracker(s, sl).setCoarseTrackingRef(fr[sl], *P[sl])
    rig.same([0, 2])
    for sl in (0, 2):
        assert out.reshape(3, 6)[sl, 0] == len(api.CoarseTracker(b, sl).cloud(0)[0])
    rig.close()


def test_map_set_batch_equals_singles():
    """reprojectMapBatch / refineBatch after sdv_map_set_batch equal them after one sdv_map_set per slot; pins follow sdv_map_set; refusals change no slot"""
    api, synth = _mods(); K, wh = synth.KITTI_K, synth.KITTI_WH
    seq = cached_sequence(6, 2000, K, wh)
    kfs_a, kfs_b = [0, 1, 2, 3], [1, 2]
    maps = [synth.make_map(seq, kfs, n_per_frame=300, seed=2 + i) for i, kfs in enumerate((kfs_a, kfs_b, kfs_a))]
    poses = np.array([np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(6)])
    kf_of = [kfs_a, kfs_b, kfs_a]; slots = [2, 0, 1]
    res = []
    for batched in (True, False):
        ctx = api.Context(K, wh[0], wh[1], n_tracker_slots=3, max_frames=8)
        for i in range(6):
            ctx.makeImages(100 + i, seq.images[i])
        rp = api.Reprojector(ctx)
        ids = [[100 + k for k in kfs] for kfs in kf_of]
        if batched:
            rp.setMapBatch(slots, ids, [m[1] for m in maps], [m[2] for m in maps], [m[0] for m in maps])
        else:
            for s, i, m in zip(slots, ids, maps):
                rp.setMap(s, i, m[1], m[2], m[0])
        cur = [105, 104, 105]
        r1 = rp.reprojectMapBatch(slots, cur, poses[[5, 4, 5]])
        r2 = rp.refineBatch(slots, cur, poses[[5, 4, 5]])
        res.append((r1, {k: v for k, v in r2.items() if k != "ms"}))
        if batched:
            assert ctx.p and api.LIB.sdv_frame_release(ctx.p, 103) == -5                          # pinned by slots 2 and 1
            rp.setMapBatch([2, 1], [[104], [104, 105]], [poses[[4]], poses[[4, 5]]], None, [maps[0][0][:0], maps[0][0][:0]])
            assert api.LIB.sdv_frame_release(ctx.p, 103) == 0                                      # the replaced slots unpinned their old keyframes
            assert api.LIB.sdv_frame_release(ctx.p, 104) == -5
            before = rp.reprojectMapBatch([0], [105], poses[[5]])
            one = np.ascontiguousarray(maps[1][0][:5])
            i32 = lambda a: np.ascontiguousarray(a, np.int32)
            call = lambda sl, hb, hf, pb: api.LIB.sdv_map_set_batch(ctx.p, len(sl), i32(sl), i32(hb), np.ascontiguousarray(hf, np.uint64), np.ascontiguousarray(np.tile(poses[1], (len(hf), 1))),
                                                                    np.zeros((len(hf), 2)), i32(pb), np.concatenate([one, one]).ctypes.data)
            assert call([0, 0], [0, 1, 2], [101, 102], [0, 5, 10]) == -1                          # a slot twice
            assert call([0, 1], [0, 1, 2], [101, 999], [0, 5, 10]) == -3                          # unknown frame (the first job would have been valid)
            assert call([0, 5], [0, 1, 2], [101, 102], [0, 5, 10]) == -1                          # slot out of range
            assert call([0, 1], [0, 0, 1], [101], [0, 5, 10]) == -1                               # a job without keyframes
            assert api.LIB.sdv_frame_release(ctx.p, 101) == -5 and api.LIB.sdv_frame_release(ctx.p, 105) == -5   # pins unchanged
            after = rp.reprojectMapBatch([0], [105], poses[[5]])
            assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0]))
        ctx.close()
    (a1, a2), (b1, b2) = res
    assert any(len(x[0]) > 10 for x in a1)
    for x, y in zip(a1, b1):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
    for k in a2:
        assert np.asarray(a2[k]).tobytes() == np.asarray(b2[k]).tobytes(), k
