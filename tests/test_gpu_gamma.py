"""GPU tests (-m gpu) of photometrically calibrated cameras at keyframe rate: sdv_set_gamma_cam (FullSystem::setGammaFunction per camera) and the gamma-weighted
absSquaredGrad of FrameHessian::makeImages that the PixelSelector reads.  Per camera, bit for bit against the oracle (orc.Frame with CalibHessian::B, pinned on the
reference's own code by tests/test_ref_pin_gamma.py): sdv_frame_download's levels and abs_out, makeHists' thresholds, makeMaps / makeMapsFromLidar maps and counts,
makeNewTraces' records (host, store and LiDAR-row forms) and the LiDAR initialiser's records and clouds, in batches that mix calibrated and uncalibrated cameras.

Context A is KITTI-360's 1400x360 at 4 levels: cameras 0-2 without gamma (1400x360, 1200x360, 1200x360), camera 3 (1200x360) with a response 255*(i/255)^0.6 and
camera 4 (1400x360) with 255*(i/1023)^1.6 over 1024 entries; twin T has the same cameras and frames and never sets a gamma.  Context B is KITTI-CARLA's 1392x1024
at 5 levels with a calibrated camera 0 and an uncalibrated 1200x360 camera at 4 levels.  A calibrated camera's frames are its raw mono8 images through
processFrame (G[v]), with a few pixels set on the x.5 rounding edges of getBGradOnly and beyond both clamps; a third frame adds intensities outside the int range
(getBGradOnly's conversion is undefined there: the x86 result, c = 5, is restated) and serves sdv_frame_download, makeHists and makeMaps only, since in makeNewTraces
such intensities make Shi-Tomasi scores NaN, whose maximum the reference and the device take differently (a property of makeNewTraces, not of the gamma)."""
import ctypes as C

import numpy as np
import pytest
import orc
import orc_gamma
import orc_init
from conftest import cached_sequence

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -5
EDGE = np.array([4.5, 5.5, 6.5, np.nextafter(np.float32(6.5), np.float32(0)), 100.5, 249.5, 250.5, 251.5, -3.0, 300.0], np.float32)
BIG = np.array([-2.5e9, 2.5e9], np.float32)                                  # outside the int range


def _mods():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth, undistort
    return api, synth, undistort


def response_text(gamma, n=256):
    """the first line of a response calibration file: 255*(i/(n-1))^gamma"""
    return " ".join(repr(float(np.float32(255.0 * (i / (n - 1)) ** gamma))) for i in range(n)) + "\n"


def photometric(text, wh, pc=2):
    _, _, U = _mods()
    return U.PhotometricUndistorter(text, np.full((wh[1], wh[0]), 200, np.uint8), wh[0], wh[1], pc)


def with_edges(img, seed, values=EDGE):
    """img with EDGE values at interior pixels of a lattice 6 px apart (away from the 4-pixel border the selector skips), each in several places.  A value outside
    the int range sits in a 3x3 patch of 128: the square roots makeHists converts to int stay in range (its (int) of a larger one is undefined in the reference).
    No NaN or inf: their arithmetic NaNs carry other bits on the GPU than on x86 (tests/test_ref_pin_gamma.py pins those on the CPU)."""
    im = np.array(img, np.float32); h, w = im.shape; rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(8, h - 8, 6), np.arange(8, w - 8, 6), indexing="ij"); pick = rng.permutation(ys.size)[:40 * len(values)]
    for (y, x), v in zip(zip(ys.reshape(-1)[pick], xs.reshape(-1)[pick]), np.tile(values, 40)):
        if abs(v) > 1e6:
            im[y - 1:y + 2, x - 1:x + 2] = 128.0
        im[y, x] = v
    return im


class World:
    """one context; camera c's frames k = 0, 1, 2 are resident as fid(c, k) (frame 2: frame 0 with BIG values too); B[c] the oracle's CalibHessian::B (None: no gamma)"""

    def __init__(self, wh, levels, cams, set_gamma=True):
        api, synth, _ = _mods(); self.api, self.synth = api, synth
        self.cams = cams; self.sizes = {c: x["wh"] for c, x in cams.items()}; self.Ks = {c: x["K"] for c, x in cams.items()}; self.levels = {c: x["L"] for c, x in cams.items()}
        self.ctx = api.Context(cams[0]["K"], *wh, levels=levels, n_tracker_slots=8, max_frames=64, max_kf_images=32)
        for c, x in cams.items():
            if c:
                self.ctx.setCameraSize(c, *x["wh"])
            if x["L"] != levels:
                self.ctx.setCameraLevels(c, x["L"])
        self.B = {}
        for c, x in cams.items():
            G = x["pu"].getG() if x.get("pu") is not None else None
            self.B[c] = None if G is None else orc_gamma.gamma_B(G)
            if set_gamma and x.get("pu") is not None:
                self.ctx.setGammaFunction(G, cam=c)
        self.images = {}
        for c, x in cams.items():
            seq = cached_sequence(2, x["seed"], x["K"], x["wh"]); self.images[(c, "seq")] = seq
            for k in range(3):
                im = seq.images[k % 2]
                if x.get("pu") is not None:                                     # what the camera's ingest makes of its raw mono8 image (processFrame)
                    im = with_edges(x["pu"].processFrame(im.astype(np.uint8)), 31 * c + k, EDGE if k < 2 else np.concatenate([EDGE, BIG]))
                self.images[(c, k)] = np.ascontiguousarray(im, np.float32)
        self.upload()
        self.rp = api.random_pattern(*wh)

    def upload(self, cams=None):
        for c in (cams or self.cams):
            ims = [self.images[(c, k)] for k in range(3)]
            self.ctx.makeImagesBatch([self.fid(c, k) for k in range(3)], [a.ctypes.data for a in ims], cams=[c] * 3)
        self.ctx.sync()

    @staticmethod
    def fid(c, k):
        return 100 * c + k + 7

    def seq(self, c):
        return self.images[(c, "seq")]

    def oframe(self, c, k, weighted=True):
        return orc_gamma.Frame(self.images[(c, k)], self.levels[c], B=self.B[c] if weighted else None)

    def orp(self, c):
        w, h = self.sizes[c]; return np.ascontiguousarray(self.rp.reshape(-1)[:w * h])


def _world_A(set_gamma=True):
    api, synth, _ = _mods(); K3 = tuple(synth.K360_K); K1 = tuple(synth.KITTI_K)
    cams = {0: dict(wh=(1400, 360), K=K3, L=4, seed=7140), 1: dict(wh=(1200, 360), K=K1, L=4, seed=7110), 2: dict(wh=(1200, 360), K=K1, L=4, seed=7111),
            3: dict(wh=(1200, 360), K=K1, L=4, seed=7112, pu=photometric(response_text(0.6), (1200, 360))),
            4: dict(wh=(1400, 360), K=K3, L=4, seed=7141, pu=photometric(response_text(1.6, 1024), (1400, 360)))}
    return World((1400, 360), 4, cams, set_gamma)


def _world_B():
    api, synth, _ = _mods()
    cams = {0: dict(wh=(1392, 1024), K=(957.962, 957.962, 696.0, 512.0), L=5, seed=7142, pu=photometric(response_text(1.6), (1392, 1024))),
            1: dict(wh=(1200, 360), K=tuple(synth.KITTI_K), L=4, seed=7110)}
    return World((1392, 1024), 5, cams)


@pytest.fixture(scope="module")
def worlds():
    A, T, B = _world_A(), _world_A(set_gamma=False), _world_B()
    yield A, T, B
    for X in (A, T, B):
        X.ctx.close()


CALIBRATED = {"A": (3, 4), "B": (0,)}


def _rows(X, ps, cams, slots, k=0):
    """LiDAR row sets of frames fid(c, k) from the front end, whose boxes are those of selector slots `slots`"""
    api, synth = X.api, X.synth; n = len(cams); fe = api.LidarFrontEnd(X.ctx)
    wl = synth.World(5100); R, t = synth.trajectory(2, 5100)
    sweeps = [synth.lidar_sweep(wl, R[k], t[k], seed=31 * j + 7 + k) for j in range(n)]
    st = fe.handleRows(list(slots), [X.fid(c, k) for c in cams], sweeps, synth.RLC, synth.TLC, np.array([X.Ks[c] for c in cams], np.float32), stats=True)
    assert all(s["rows"] > 300 and not s["overflow"] for s in st)
    return [fe.rows(X.fid(c, k)) for c in cams]


MAPS = ((600.0, 1, 1.0, 0), (3000.0, 1, 2.0, 2), (150.0, 0, 1.0, 2))    # density, recursionsLeft, thFactor, frame of three makeMaps rounds


def _lrud(q):
    return np.array([int(q[:, 0].min()), int(q[:, 0].max()), int(q[:, 1].min()), int(q[:, 1].max())], np.int32)


def device_results(X, cams):
    """everything the keyframe-rate path computes for frames of `cams`, one batch mixing all of them per stage, per camera.  Selector slots: [0, n) makeMapsFromLidar,
    [n, 2n) makeMaps, [2n, 3n) makeNewTraces, [3n, 4n) its store form, [4n, 5n) the LiDAR-row form, [5n, 6n) the store form fed those rows."""
    api = X.api; n = len(cams); out = {c: {} for c in cams}
    for c in cams:
        for k in range(3):
            for l in range(X.levels[c]):
                dI, ab = X.ctx.frameLevel(X.fid(c, k), l); out[c][f"dI{k}{l}"] = dI.tobytes(); out[c][f"abs{k}{l}"] = ab.tobytes()
        ps = api.PixelSelector(X.ctx, 1, X.rp, cams=[c])
        for k in (0, 2):
            out[c][f"hists{k}"] = b"".join(a.tobytes() for a in ps.makeHists(X.fid(c, k), cam=c))
    ps = api.PixelSelector(X.ctx, 6 * n, X.rp, cams=list(cams) * 6); sl = lambda q: list(range(q * n, (q + 1) * n))
    frames = [X.fid(c, 0) for c in cams]; clouds = [X.seq(c).clouds[0] for c in cams]
    for rnd, (dens, rec, th, k) in enumerate(MAPS):
        mL, nL = ps.makeMapsBatch(sl(0), [X.fid(c, k) for c in cams], dens, rec, th, clouds=clouds)
        mD, nD = ps.makeMapsBatch(sl(1), [X.fid(c, k) for c in cams], dens, rec, th)
        for j, c in enumerate(cams):
            out[c][f"mapsL{rnd}"] = (mL[j].tobytes(), int(nL[j]), ps.potential(j)); out[c][f"mapsD{rnd}"] = (np.asarray(mD[j]).tobytes(), int(nD[j]), ps.potential(n + j))
    S = api.ImmatureStore(X.ctx)
    for k in range(2):
        fr = [X.fid(c, k) for c in cams]; cl = [X.seq(c).clouds[k] for c in cams]
        dl = [api.lidar_density(_lrud(cl[j]), X.sizes[c], 900.0) for j, c in enumerate(cams)]
        res, num = ps.makeNewTracesBatch(sl(2), fr, cl, dl, 900.0, 1, cap=1 << 15)
        n_s, num_s = ps.makeNewTracesStore(sl(3), fr, cl, dl, 900.0, 1, cap=1 << 15)
        assert np.array_equal(num, num_s) and [len(r[0]) for r in res] == n_s.tolist()
        for j, c in enumerate(cams):
            g, m = S.get(fr[j]); P, M = _after_make_key_frame(api, *res[j])
            assert g.tobytes() == P.tobytes() and m.tobytes() == M.tobytes(), (k, c)
            out[c][f"traces{k}"] = (res[j][0].tobytes(), res[j][1].tobytes(), num[j].tolist(), ps.selectionMap(2 * n + j).tobytes())
        S.drop(fr)
    # the LiDAR-row form: rows, box and addFeaturePoint of each frame's set, against the store form fed the same rows
    rows = _rows(X, ps, cams, sl(4))
    n_r, num_r = ps.makeNewTracesRowsStore(sl(4), frames, 900.0, cap=1 << 15); blocks = [S.get(f) for f in frames]
    dl = [api.lidar_density(rows[j]["lrud"], X.sizes[c], 900.0) for j, c in enumerate(cams)]
    n_h, num_h = ps.makeNewTracesStore(sl(5), frames, [r["cloud_px"] for r in rows], dl, 900.0, [r["addFeaturePoint"] for r in rows], cap=1 << 15)
    assert np.array_equal(n_r, n_h) and np.array_equal(num_r, num_h)
    for j, c in enumerate(cams):
        g, m = S.get(frames[j]); assert g.tobytes() == blocks[j][0].tobytes() and m.tobytes() == blocks[j][1].tobytes(), c
        out[c]["rows_traces"] = (blocks[j][0].tobytes(), blocks[j][1].tobytes(), num_r[j].tolist())
    S.drop(frames)
    # the LiDAR initialiser from the same row sets (sdv_init_from_lidar_rows_batch), on tracker slots 0..n-1 bound to the cameras
    X.ctx.setCalibSlots(list(range(n)), [X.Ks[c] for c in cams], cams=list(cams))
    draws = [np.random.default_rng(5 + j).integers(0, 2**31 - 1, len(r["cloud_px"])).astype(np.int32) for j, r in enumerate(rows)]
    res = api.initializeFromLidarBatch(X.ctx, list(range(n)), frames, None, None, [300.0 + 200 * j for j in range(n)], draws)
    for j, c in enumerate(cams):
        tr = api.CoarseTracker(X.ctx, j)
        out[c]["init"] = (int(res["n_selected"][j]), res["pts"][j].tobytes(), res["meta"][j].tobytes(), res["idepth"][j].tobytes(),
                          [np.stack(tr.cloud(l), 1).tobytes() for l in range(X.levels[c])])
    return out, dict(rows=rows, draws=draws)


def _after_make_key_frame(api, T, I):
    from test_gpu_immature_store import _after_make_key_frame as f
    return f(api, T, I)


def oracle_results(X, cams, aux, weighted=True):
    """the same from the oracle (orc.Frame with the camera's B), with NEW oracle selector state per slot as the device's slots start"""
    api = X.api; n = len(cams); out = {c: {} for c in cams}
    of = {(c, k): X.oframe(c, k, weighted) for c in cams for k in range(3)}
    for c in cams:
        w, h = X.sizes[c]
        for k in range(3):
            for l in range(X.levels[c]):
                out[c][f"dI{k}{l}"] = of[(c, k)].dI(l).tobytes(); out[c][f"abs{k}{l}"] = of[(c, k)].absSquaredGrad(l).tobytes()
        for k in (0, 2):
            out[c][f"hists{k}"] = b"".join(a.tobytes() for a in orc.Selector(w, h, X.orp(c)).makeHists(of[(c, k)]))
        sL, sD = orc.Selector(w, h, X.orp(c)), orc.Selector(w, h, X.orp(c))
        for rnd, (dens, rec, th, k) in enumerate(MAPS):
            m, num = sL.makeMaps(of[(c, k)], dens, rec, th, X.seq(c).clouds[0]); out[c][f"mapsL{rnd}"] = (m.astype(np.uint8).tobytes(), int(num), sL.currentPotential)
            m, num = sD.makeMaps(of[(c, k)], dens, rec, th, None); out[c][f"mapsD{rnd}"] = (m.astype(np.uint8).tobytes(), int(num), sD.currentPotential)
        sN = orc.Selector(w, h, X.orp(c)); sel = np.zeros((h, w), np.float32)
        for k in range(2):
            q = X.seq(c).clouds[k]
            T, num, _ = sN.makeNewTraces(of[(c, k)], q, orc.lidar_density(_lrud(q), (w, h), 900.0), 900.0, 1, sel)
            out[c][f"traces{k}"] = T
        j = cams.index(c); r = aux["rows"][j]
        sR = orc.Selector(w, h, X.orp(c)); T, num, _ = sR.makeNewTraces(of[(c, 0)], r["cloud_px"], orc.lidar_density(r["lrud"], (w, h), 900.0), 900.0, r["addFeaturePoint"], np.zeros((h, w), np.float32))
        out[c]["rows_traces"] = T
        ot = orc.CoarseTracker(w, h, X.levels[c], X.Ks[c])
        o = orc_init.init_from_lidar(of[(c, 0)], X.orp(c), r["cloud_px"], r["lrud"], 300.0 + 200 * j, aux["draws"][j], tracker=ot)
        out[c]["init"] = (int(o["n_selected"]), o["pts"].tobytes(), o["meta"].tobytes(), o["idepth"].tobytes(), [np.stack(ot.cloud(l), 1).tobytes() for l in range(X.levels[c])])
    return out


def _same_as_oracle(dev, orc_, c):
    """device results of camera c equal the oracle's: arrays bit for bit, makeNewTraces records as the oracle's NEW_TRACE rows"""
    d, o = dev[c], orc_[c]
    for key in d:
        if key.startswith("traces"):
            assert d[key][0] == o[key].tobytes(), (c, key)
        elif key == "rows_traces":                                      # the store's records and meta against the oracle's NEW_TRACE rows
            api = _mods()[0]; P = np.frombuffer(d[key][0], dtype=api.IMMATURE_PT_DTYPE); M = np.frombuffer(d[key][1], dtype=api.IMMATURE_META_DTYPE); T = o[key]
            assert len(P) == len(T) and np.array_equal(P["u"], T["u"]) and np.array_equal(P["v"], T["v"]), c
            assert all(np.array_equal(M[f], T[f]) for f in ("my_type", "type", "isFromSensor", "idepth_fromSensor")), c
        else:
            assert d[key] == o[key], (c, key)


def test_calibrated_and_plain_cameras_match_oracle(worlds):
    """context A (1400x360 and 1200x360 cameras, two calibrated) and context B (1392x1024 at 5 levels calibrated, 1200x360 plain): every stage, one mixed batch
    per stage, equals the oracle with each camera's B; on a calibrated camera the weighted result differs from the unweighted one at every stage"""
    A, T, B = worlds
    for name, X in (("A", A), ("B", B)):
        cams = list(X.cams); dev, aux = device_results(X, cams); o = oracle_results(X, cams, aux)
        for c in cams:
            _same_as_oracle(dev, o, c)
        plain = oracle_results(X, list(CALIBRATED[name]), dict(rows=[aux["rows"][cams.index(c)] for c in CALIBRATED[name]],
                                                              draws=[aux["draws"][cams.index(c)] for c in CALIBRATED[name]]), weighted=False)
        for c in CALIBRATED[name]:
            d, p = dev[c], plain[c]
            assert all(d[f"dI{k}{l}"] == p[f"dI{k}{l}"] for k in range(3) for l in range(X.levels[c])), c           # the gradients are unweighted
            assert all(d[f"abs{k}{l}"] != p[f"abs{k}{l}"] for k in range(3) for l in range(X.levels[c])), c
            assert d["hists0"] != p["hists0"] and d["hists2"] != p["hists2"], c
            assert all(d[f"maps{t}{r}"][0] != p[f"maps{t}{r}"][0] for t in "LD" for r in range(3)), c
            assert d["traces0"][0] != p["traces0"].tobytes() and d["traces1"][0] != p["traces1"].tobytes(), c
            assert d["init"][1] != p["init"][1], c


def test_uncalibrated_cameras_unchanged(worlds):
    """cameras 0-2 of context A give exactly what a context that never called sdv_set_gamma_cam gives, in the same mixed batches"""
    A, T, B = worlds
    cams = list(A.cams); da, _ = device_results(A, cams); dt, _ = device_results(T, cams)
    for c in (0, 1, 2):
        assert da[c] == dt[c], c
    for c in CALIBRATED["A"]:
        assert da[c]["abs00"] != dt[c]["abs00"] and da[c]["traces0"] != dt[c]["traces0"], c


def test_identity_and_null_change_nothing():
    """the identity response, the linearised 256-entry response of main.cpp's modes 1 and 2 (setting_photometricCalibration = 0), a gamma reset with NULL and
    a non-increasing response (invalid: getG() is None) all give what no gamma gives"""
    import types
    api, synth, U = _mods()
    T = _world_A(set_gamma=False); X = _world_A(set_gamma=False)
    try:
        bad = " ".join(str(v) for v in list(range(100)) + [99] + list(range(100, 255))) + "\n"
        for c in X.cams:
            for k in range(3):
                X.ctx.releaseFrame(X.fid(c, k))
        X.ctx.setGammaFunction(np.arange(256, dtype=np.float32), cam=0)
        for c, text, pc in ((1, response_text(0.6), 0), (3, bad, 2)):                       # mode 1 / 2: linearised G; an invalid calibration
            w, h = X.sizes[c]; pu = photometric(text, (w + 2, h + 2), pc); x, y = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
            und = types.SimpleNamespace(wOrg=w + 2, hOrg=h + 2, remapX=x + 1, remapY=y + 1, G=pu.ingest_G, vignetteMapInv=pu.ingest_vignetteMapInv, photometricUndist=pu)
            assert (pu.getG() is None) == (c == 3) and pu.ingest_G is None
            X.ctx.setCameraPhotometric(und, cam=c)
        X.ctx.setGammaFunction(photometric(response_text(0.6), (10, 10)).getG(), cam=2); X.ctx.setGammaFunction(None, cam=2)
        X.ctx.setGammaFunction(None, cam=4)
        X.upload()
        cams = list(X.cams); dx, _ = device_results(X, cams); dt, _ = device_results(T, cams)
        for c in cams:
            assert dx[c] == dt[c], c
    finally:
        T.ctx.close(); X.ctx.close()


def test_refusals_leave_the_tables():
    """a resident frame of the camera (SDV_ERR_STATE), a camera out of range and a NULL context (SDV_ERR_ARG) change no table: the frames ingested after the
    refusals carry the weights of the gamma set before them"""
    api, synth, U = _mods(); X = _world_A()
    try:
        L = api.LIB; G = photometric(response_text(1.6), (10, 10)).getG(); g = np.ascontiguousarray(G[:256], np.float32)
        for c in X.cams:
            assert L.sdv_set_gamma_cam(X.ctx.p, c, g.ctypes.data) == ERR_STATE, c
            assert L.sdv_set_gamma_cam(X.ctx.p, c, None) == ERR_STATE, c
        for c in (-1, 8, 99):
            assert L.sdv_set_gamma_cam(X.ctx.p, c, g.ctypes.data) == ERR_ARG, c
        assert L.sdv_set_gamma_cam(None, 3, g.ctypes.data) == ERR_ARG and L.sdv_set_gamma_cam(None, 3, None) == ERR_ARG
        with pytest.raises(api.SdvError):
            X.ctx.setGammaFunction(G, cam=3)
        for c in X.cams:
            for k in range(3):
                X.ctx.releaseFrame(X.fid(c, k))
        X.upload()
        for c in X.cams:
            for l in range(X.levels[c]):
                _, ab = X.ctx.frameLevel(X.fid(c, 2), l)
                assert ab.tobytes() == X.oframe(c, 2).absSquaredGrad(l).tobytes(), (c, l)
    finally:
        X.ctx.close()
