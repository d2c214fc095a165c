"""GPU tests (-m gpu) of the start of a sequence on the device: sdv_init_from_lidar_batch (host rows) and sdv_init_from_lidar_rows_batch (LiDAR row sets) —
CoarseInitializer::setFirstFromLidar at level 0, the point loop of FullSystem::initializeFromInitializer and setCTRefForFirstFrame, with the tracker reference and the
one-keyframe map installed on the device.  Records, numPoints[0], points kept and the slot clouds must equal the oracle (oracle/orc_init.cpp, pinned on the
reference's own code by tests/test_ref_pin_init.py) bit for bit, in both forms, for a batch of cameras of different sizes and depths.

Context A is KITTI-360's 1400x360 at 4 levels with a KITTI 1200x360 camera and a 1244x356 camera; context B is KITTI-CARLA's 1392x1024 at 5 levels with a
KITTI 1200x360 camera at 4 levels."""
import ctypes as C

import numpy as np
import pytest
import orc
import orc_init
from conftest import cached_sequence

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_NOFRAME, ERR_CAPACITY, ERR_STATE = -1, -3, -4, -5
T0 = np.array([1, 0, 0, 0, 0, 0, 0.0])


def _mods():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    return api, synth


class Ctx:
    """one context; sequence j runs on camera cams[j] and on selector / tracker / map slot j; its frames k = 0, 1 are resident under handle fid(j, k)"""

    def __init__(self, wh, levels, cams, extra):
        api, synth = _mods(); self.api, self.synth = api, synth
        self.sizes = {0: wh}; self.levels = {0: levels}; self.Ks = {0: extra[0][1]}; seeds = {c: e[3] for c, e in enumerate(extra)}
        self.ctx = api.Context(extra[0][1], *wh, levels=levels, n_tracker_slots=8, max_frames=64, max_kf_images=16)
        for c, (sz, K, L, _) in enumerate(extra[1:], start=1):
            self.ctx.setCameraSize(c, *sz); self.sizes[c] = sz; self.Ks[c] = K
            if L != levels:
                self.ctx.setCameraLevels(c, L)
            self.levels[c] = L
        self.cams = list(cams); n = len(cams)
        self.seqs = [cached_sequence(2, seeds[c], self.Ks[c], self.sizes[c]) for c in self.cams]
        for j, c in enumerate(self.cams):
            ims = [np.ascontiguousarray(im, np.float32) for im in self.seqs[j].images[:2]]
            self.ctx.makeImagesBatch([self.fid(j, k) for k in range(2)], [a.ctypes.data for a in ims], cams=[c] * 2)
        self.ctx.sync()
        self.rp = api.random_pattern(*wh)
        self.ps = api.PixelSelector(self.ctx, n, self.rp, cams=self.cams)
        self.ctx.setCalibSlots(list(range(n)), [self.Ks[c] for c in self.cams], cams=self.cams)
        self.fe = api.LidarFrontEnd(self.ctx)
        wl = synth.World(5100); R, t = synth.trajectory(2, 5100)
        sweeps = [synth.lidar_sweep(wl, R[0], t[0], seed=31 * j + 7) for j in range(n)]
        st = self.fe.handleRows(list(range(n)), [self.fid(j, 0) for j in range(n)], sweeps, synth.RLC, synth.TLC,
                                np.array([self.Ks[c] for c in self.cams], np.float32), stats=True)
        assert all(s["rows"] > 500 and not s["overflow"] for s in st)
        self.rows = [self.fe.rows(self.fid(j, 0)) for j in range(n)]

    @staticmethod
    def fid(j, k):
        return 1000 + 10 * j + k

    def L(self, j):
        return self.levels[self.cams[j]]

    def wh(self, j):
        return self.sizes[self.cams[j]]

    def oracle(self, j, cloud, lrud, density, draws):
        w, h = self.wh(j); f0 = orc.Frame(self.seqs[j].images[0], self.L(j)); ot = orc.CoarseTracker(w, h, self.L(j), self.Ks[self.cams[j]])
        return orc_init.init_from_lidar(f0, self.rp, cloud, lrud, density, draws, tracker=ot), ot, f0

    def clouds(self, j):
        tr = self.api.CoarseTracker(self.ctx, j)
        return [np.stack(tr.cloud(l), 1) for l in range(self.L(j))]


@pytest.fixture(scope="module")
def ctxs():
    api, synth = _mods()
    K3 = (702.5, 698.0, 611.0, 171.5)
    # per camera: size, K, depth, seed of its synthetic drive (drives whose first two frames the tracker follows from the identity hypothesis)
    A = Ctx((1400, 360), 4, [0, 1, 2, 1], [(None, tuple(synth.K360_K), 4, 7140), ((1200, 360), tuple(synth.KITTI_K), 4, 7110), ((1244, 356), K3, 4, 7120)])
    B = Ctx((1392, 1024), 5, [0, 1], [(None, (957.962, 957.962, 696.0, 512.0), 5, 7140), ((1200, 360), tuple(synth.KITTI_K), 4, 7110)])
    yield A, B
    A.ctx.close(); B.ctx.close()


DENS = [300.0, 1e6, 700.0, 150.0]


def _draws(X, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 2**31 - 1, size=len(r["cloud_px"]), dtype=np.int64).astype(np.int32) for r in X.rows]


def _check_vs_oracle(X, j, res, jj, density, draws):
    o, ot, _ = X.oracle(j, X.rows[j]["cloud_px"], X.rows[j]["lrud"], density, draws)
    assert res["n_selected"][jj] == o["n_selected"] and res["n"][jj] == len(o["pts"]), (j, res["n_selected"][jj], o["n_selected"])
    assert res["pts"][jj].tobytes() == o["pts"].tobytes() and res["meta"][jj].tobytes() == o["meta"].tobytes() and np.array_equal(res["idepth"][jj], o["idepth"]), j
    for l, g in enumerate(X.clouds(j)):
        assert g.tobytes() == np.stack(ot.cloud(l), 1).tobytes(), (j, l)
    return o


@pytest.mark.parametrize("form", ["rows", "host"])
def test_batch_matches_oracle(ctxs, form):
    """three camera sizes in one 1400x360 context, a 5-level camera beside a 4-level one in a 1392x1024 context: both entry forms equal the oracle bit for bit"""
    for X in ctxs:
        api = X.api; n = len(X.cams); dens = DENS[:n]; dr = _draws(X, 1)
        clouds = None if form == "rows" else [r["cloud_px"] for r in X.rows]; lr = None if form == "rows" else [r["lrud"] for r in X.rows]
        res = api.initializeFromLidarBatch(X.ctx, list(range(n)), [X.fid(j, 0) for j in range(n)], clouds, lr, dens, dr)
        for j in range(n):
            o = _check_vs_oracle(X, j, res, j, dens[j], dr[j])
            assert o["n_selected"] > 50 and len(o["pts"]) > 20
            assert dens[j] > 1e5 or len(o["pts"]) < o["n_selected"]


def test_batching_is_invisible(ctxs):
    """a batch equals its jobs called one by one, and the same call twice gives the same records and clouds"""
    X = ctxs[0]; api = X.api; n = len(X.cams); dr = _draws(X, 2); frames = [X.fid(j, 0) for j in range(n)]
    one = [api.initializeFromLidarBatch(X.ctx, [j], [frames[j]], None, None, DENS[j], [dr[j]]) for j in range(n)]
    cl_one = [X.clouds(j) for j in range(n)]
    for rep in range(2):
        res = api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, None, None, DENS[:n], dr)
        for j in range(n):
            assert res["n"][j] == one[j]["n"][0] and res["n_selected"][j] == one[j]["n_selected"][0]
            for k in ("pts", "meta", "idepth"):
                assert res[k][j].tobytes() == one[j][k][0].tobytes(), (rep, j, k)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(X.clouds(j), cl_one[j])), (rep, j)


def test_installed_state_equals_existing_entries(ctxs):
    """the slot's clouds equal sdv_tracker_set_ref fed the returned records ({u, v, idepth, 0}, round_half 1); the map gives the reprojectMap matches on frame 1
    that sdv_map_set of the records gives"""
    X = ctxs[0]; api = X.api; n = len(X.cams); dr = _draws(X, 3); frames = [X.fid(j, 0) for j in range(n)]
    res = api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, None, None, DENS[:n], dr)
    rp = api.Reprojector(X.ctx); cur = [X.fid(j, 1) for j in range(n)]
    T1 = np.stack([np.concatenate([X.synth._quat_from_R(X.seqs[j].R[1]), X.seqs[j].t[1]]) for j in range(n)])
    T1 = np.stack([orc.se3_mul(orc.se3_inv(np.concatenate([X.synth._quat_from_R(X.seqs[j].R[0]), X.seqs[j].t[0]])), T1[j]) for j in range(n)])
    dev_clouds = [X.clouds(j) for j in range(n)]; dev_match = rp.reprojectMapBatch(list(range(n)), cur, T1)
    assert sum(len(m[0]) for m in dev_match) > 50
    for j in range(n):
        P = res["pts"][j]; d = res["idepth"][j]
        pts4 = np.stack([P["u"], P["v"], d, np.zeros(len(P), np.float32)], 1)
        api.CoarseTracker(X.ctx, j).setCoarseTrackingRef(frames[j], pts4, np.ones(len(P), np.int32))
        mp = np.zeros(len(P), api.MAP_PT_DTYPE); mp["u"], mp["v"], mp["idepth"] = P["u"], P["v"], d
        rp.setMap(j, [frames[j]], T0.reshape(1, 7), np.zeros((1, 2)), mp)
    host_match = rp.reprojectMapBatch(list(range(n)), cur, T1)
    for j in range(n):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(X.clouds(j), dev_clouds[j])), j
        assert dev_match[j][0].tobytes() == host_match[j][0].tobytes() and dev_match[j][1].tobytes() == host_match[j][1].tobytes(), j


def test_frame_one_follows(ctxs):
    """sdv_track_new_coarse_batch with poses_valid = 2 after the device bootstrap against the oracle's trackNewCoarse after the oracle's bootstrap.  The bootstrap
    state is the oracle's bit for bit (the records here, the clouds and the map in the tests above); the tracker's float sums then run in another order than the
    oracle's (test_gpu_slot_calib.py), so the LM lands within rounding of the oracle's pose rather than on it: same tries, winner and match count, energies within
    1e-4 relative, poses within 1e-3 m / rad.  The rows are the drives' own LiDAR pixels (host form), the draws the C library's stream of a running reference."""
    for X in ctxs:
        api = X.api; n = len(X.cams); frames = [X.fid(j, 0) for j in range(n)]
        clouds = [X.seqs[j].clouds[0] for j in range(n)]
        lr = [np.array([int(c[:, 0].min()), int(c[:, 0].max()), int(c[:, 1].min()), int(c[:, 1].max())], np.int32) for c in clouds]
        dr = [api.initializer_draws(*X.wh(j), len(clouds[j])) for j in range(n)]
        res = api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, clouds, lr, 1500.0, dr)
        jobs = [dict(slot=j, frame=X.fid(j, 1), poses_valid=2, sprelast_c2w=T0, slast_c2w=T0, lastF_c2w=T0, aff_last=[0.0, 0.0], lastCoarseRMSE=[100.0] * 5) for j in range(n)]
        g = api.trackNewCoarseBatch(X.ctx, jobs)
        for j in range(n):
            o, ot, f0 = X.oracle(j, clouds[j], lr[j], 1500.0, dr[j])
            assert res["n"][j] == len(o["pts"]) and res["pts"][j].tobytes() == o["pts"].tobytes()
            mp = np.zeros(len(o["pts"]), api.MAP_PT_DTYPE); mp["u"], mp["v"], mp["idepth"] = o["pts"]["u"], o["pts"]["v"], o["idepth"]
            f1 = orc.Frame(X.seqs[j].images[1], X.L(j))
            r = orc.track_new_coarse(ot, f1, X.Ks[X.cams[j]], [f0], T0.reshape(1, 7), np.zeros((1, 2)), mp, T0, T0, T0, [0.0, 0.0], 2, np.full(5, 100.0))
            assert (g[j]["tries"], g[j]["have_one_good"], g[j]["n_matches"]) == (r["tries"], r["have_one_good"], r["n_matches"]) and r["have_one_good"], j
            assert np.allclose(g[j]["lastCoarseRMSE"], r["lastCoarseRMSE"], rtol=1e-4, equal_nan=True), j
            assert np.abs(orc.se3_log(orc.se3_mul(np.asarray(g[j]["camToTrackingRef"]), orc.se3_inv(r["camToTrackingRef"])))).max() < 1e-3, j


def test_reference_run_follows():
    """the reference's own FullSystem over the first two frames of S-KITTI-200 (tests/golden/seq_init_ref.npz): the device bootstrap of frame 0 and the
    53-hypothesis trackNewCoarse of frame 1 give its numPoints[0], its pose within 1e-3 m / 1e-3 rad and its energy within 1e-4 relative"""
    api, synth = _mods()
    from test_ref_pin_init import reference_start
    g, seq, draws, order = reference_start(); w, h = seq.wh; K = tuple(synth.KITTI_K)
    ctx = api.Context(K, w, h, levels=int(g["levels"]), max_frames=4, affineOptModeA=-1.0, affineOptModeB=-1.0)     # mode 2 of main.cpp:461-468, as the reference run
    try:
        for k in range(2):
            ctx.makeImages(k, np.ascontiguousarray(seq.images[k], np.float32))
        api.PixelSelector(ctx, 1, api.random_pattern(w, h))
        res = api.initializeFromLidarBatch(ctx, [0], [0], [g["rows0"]], [g["lrud0"]], 1500.0, [draws])
        assert res["n_selected"][0] == int(g["n_selected"])
        r = api.trackNewCoarseBatch(ctx, [dict(slot=0, frame=1, poses_valid=2, sprelast_c2w=T0, slast_c2w=T0, lastF_c2w=T0, aff_last=[0.0, 0.0], lastCoarseRMSE=[100.0] * 5)],
                                    cell_order=order)[0]
        d = orc.se3_log(orc.se3_mul(r["camToTrackingRef"], orc.se3_inv(g["camToTrackingRef"])))
        assert np.abs(d).max() < 1e-3, d
        assert abs(r["lastCoarseRMSE"][0] - g["lastCoarseRMSE"][0]) <= 1e-4 * g["lastCoarseRMSE"][0], (r["lastCoarseRMSE"], g["lastCoarseRMSE"])
        assert np.allclose(r["aff_g2l"], g["aff_g2l"], atol=1e-9)
    finally:
        ctx.close()


def _slot_state(X, n):
    """everything the call must not touch and every slot a refused call must leave alone"""
    api = X.api; st = [X.ps.potential(s) for s in range(n)] + [X.ps.selectionMap(s).tobytes() for s in range(n)] + [X.ps.lidarBox(s).tolist() for s in range(n)]
    cnt = np.zeros(1, np.int32)
    st += [api.LIB.sdv_immature_store_count(X.ctx.p, 1, np.array([X.fid(j, 0)], np.uint64), cnt) for j in range(n)]
    st += [b"".join(c.tobytes() for c in X.clouds(j)) for j in range(n)]
    m = api.Reprojector(X.ctx).reprojectMapBatch(list(range(n)), [X.fid(j, 1) for j in range(n)], np.tile(T0, (n, 1)))
    return st + [a.tobytes() + b.tobytes() for a, b in m]


def _rc(X, slots, frames, draws, cap=1 << 14, rows=True, clouds=None, lruds=None):
    api = X.api; n = len(slots); dr = [np.ascontiguousarray(d, np.int32) for d in draws]
    db = np.concatenate([[0], np.cumsum([len(d) for d in dr])]).astype(np.int32); da = np.ascontiguousarray(np.concatenate(dr + [np.zeros(1, np.int32)]))
    o = [np.zeros(max(n, 1), np.int32) for _ in range(2)]; dens = np.full(n, 500.0, np.float32)
    if rows:
        rc = api.LIB.sdv_init_from_lidar_rows_batch(X.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frames, np.uint64), dens, db, da, cap, o[0], o[1], None, None, None)
    else:
        cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; cb = np.concatenate([[0], np.cumsum([len(c) for c in cl])]).astype(np.int32)
        c3 = np.ascontiguousarray(np.concatenate(cl + [np.zeros((1, 3))])); box = np.ascontiguousarray(lruds, np.int32).reshape(-1)
        rc = api.LIB.sdv_init_from_lidar_batch(X.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frames, np.uint64), cb, c3.ctypes.data, box, dens, db, da,
                                               cap, o[0], o[1], None, None, None)
    return rc, o[0][:n], o[1][:n]


def test_nothing_else_is_touched_and_refusals(ctxs):
    """selector slots (potential, map, box) and the immature store are the same after the call; every refusal returns its code before anything is enqueued and leaves
    the tracker and map slots as they were; an empty cloud gives a reference of 0 points at every level"""
    X = ctxs[0]; api = X.api; n = len(X.cams); dr = _draws(X, 4); frames = [X.fid(j, 0) for j in range(n)]
    X.ps.potential(1, set_to=5); X.ps.makeMapsBatch([0], [frames[0]], 800.0)        # selector slots with state of their own
    synth = X.synth; wl = synth.World(5100); R, t = synth.trajectory(2, 5100)                    # an overflowed row set: more pixel rows than its cap
    X.fe.handleRows([3], [4343], [synth.lidar_sweep(wl, R[1], t[1], seed=5)], synth.RLC, synth.TLC, np.array([X.Ks[X.cams[3]]], np.float32), cap=10, stats=True)
    api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, None, None, DENS[:n], dr)
    before = _slot_state(X, n)
    api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, None, None, DENS[:n], dr)
    assert _slot_state(X, n) == before
    cases = [
        (ERR_NOFRAME, dict(slots=[0, 1], frames=[frames[0], 4242], draws=dr[:2])),                                              # no row set
        (ERR_ARG, dict(slots=[0, 1], frames=frames[:2], draws=[dr[0], dr[1][:-1]])),                                            # too few draws
        (ERR_ARG, dict(slots=[0, n], frames=frames[:2], draws=dr[:2])),                                                         # slot out of range
        (ERR_ARG, dict(slots=[1, 1], frames=frames[:2], draws=dr[:2])),                                                         # slot twice
        (ERR_ARG, dict(slots=[0, 1], frames=[frames[1], frames[1]], draws=[dr[1], dr[1]])),                                     # frame twice
        (ERR_ARG, dict(slots=[0, 1], frames=[frames[1], frames[0]], draws=[dr[1], dr[0]])),                                     # a 1200x360 frame on a 1400x360 slot
        (ERR_CAPACITY, dict(slots=[0, 1], frames=frames[:2], draws=dr[:2], cap=5)),                                             # more kept points than cap
    ]
    for code, kw in cases:
        rc, n_out, n_sel = _rc(X, kw["slots"], kw["frames"], kw["draws"], cap=kw.get("cap", 1 << 14))
        assert rc == code, (code, kw["slots"], kw["frames"], api.LIB.sdv_last_error(X.ctx.p))
        if code == ERR_CAPACITY:
            assert n_out[0] > 5 and n_sel[0] >= n_out[0]
        assert _slot_state(X, n) == before, code
    assert _rc(X, [0, 3], [frames[0], 4343], [dr[0], np.zeros(20000, np.int32)])[0] == ERR_CAPACITY
    assert _slot_state(X, n) == before
    # no selector engine
    Y = api.Context(X.Ks[0], *X.sizes[0], levels=4, max_frames=4); Y.makeImages(7, np.ascontiguousarray(X.seqs[0].images[0], np.float32))
    o = [np.zeros(1, np.int32) for _ in range(2)]
    rc = api.LIB.sdv_init_from_lidar_batch(Y.p, 1, np.zeros(1, np.int32), np.array([7], np.uint64), np.zeros(2, np.int32), None, np.array([0, 1, 0, 1], np.int32),
                                          np.ones(1, np.float32), np.zeros(2, np.int32), np.zeros(1, np.int32), 16, o[0], o[1], None, None, None)
    assert rc == ERR_STATE; Y.close()
    # the empty cloud: no point kept, 0 points at every level, a map of one keyframe and no point
    rc, n_out, n_sel = _rc(X, [0], [frames[0]], [np.zeros(1, np.int32)], rows=False, clouds=[np.zeros((0, 3))], lruds=[[10000, -1, 10000, -1]])
    assert rc == 0 and n_out[0] == 0 and n_sel[0] == 0
    assert all(len(c) == 0 for c in X.clouds(0))
    assert len(api.Reprojector(X.ctx).reprojectMap(0, X.fid(0, 1), T0)[0]) == 0
