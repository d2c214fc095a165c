"""GPU tests (-m gpu) of the LiDAR row sets: lidarCloudHandler writing its pixel rows into device-resident sets keyed by frame handle
(sdv_lidar_handler_rows_batch), the running pixel box kept per selector slot on the device, and makeNewTraces fed from the sets into the immature-point store
(sdv_make_new_traces_rows_store_batch).  Every result must equal, bit for bit, the host-row path (sdv_lidar_handler_batch_cams with the host carrying the box,
sdv_make_new_traces_store_batch fed the downloaded rows) and the oracle (pinned on the reference's own main.cpp).

Two contexts of KITTI-360's size 1400x360 with a KITTI 1200x360 camera and a 1244x356 camera hold the same six sequences (test_gpu_immature_store.World):
context A runs the row-set path, context B the host-row path."""
import ctypes as C
import numpy as np
import pytest
import orc
from test_gpu_immature_store import World, MIX, DENS, SIZES, fid, _window

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_NOFRAME, ERR_CAPACITY, ERR_STATE = -1, -3, -4, -5
BOX0 = [10000, -1, 10000, -1]


@pytest.fixture(scope="module")
def worlds():
    a, b = World(), World()
    yield a, b
    a.ctx.close(); b.ctx.close()


def _sweeps(W, k, upper=()):
    """one raw sweep per sequence for frame k (mostly ground: addFeaturePoint 1); jobs in `upper` keep only returns above z = -1.4 m (addFeaturePoint 0)"""
    synth = W.synth; wl = synth.World(5100); R, t = synth.trajectory(6, 5100)
    S = [synth.lidar_sweep(wl, R[k % 6], t[k % 6], seed=10 * j + k) for j in range(len(MIX))]
    return [s[s[:, 2] > -1.4] if j in upper else s for j, s in enumerate(S)]


def _K4(W, cams=MIX):
    return np.array([W.Ks[c] for c in cams], np.float32)


def _rows_rc(W, slots, frames, sweeps, cams, cap=1 << 15, tlc=None):
    """sdv_lidar_handler_rows_batch called directly -> return code"""
    api, synth = W.api, W.synth; n = len(slots)
    sw = [np.ascontiguousarray(s, np.float32).reshape(-1, 4) for s in sweeps]; sb = np.concatenate([[0], np.cumsum([len(s) for s in sw])]).astype(np.int32)
    allp = np.ascontiguousarray(np.concatenate(sw)); R = np.ascontiguousarray(np.tile(synth.RLC.reshape(-1), n), np.float64)
    t = np.ascontiguousarray(np.tile(np.asarray(synth.TLC if tlc is None else tlc, np.float64), n)); K = np.ascontiguousarray(_K4(W, cams).reshape(-1))
    return api.LIB.sdv_lidar_handler_rows_batch(W.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frames, np.uint64), sb, allp.ctypes.data, R, t, K, cap, None)


def _state(W, ps, fe, n_slots, frames):
    """everything a refused call must leave alone: boxes, potentials, maps, row sets, store blocks"""
    S = W.api.ImmatureStore(W.ctx); out = [ps.lidarBox(s).tolist() for s in range(n_slots)] + [ps.potential(s) for s in range(n_slots)]
    out += [ps.selectionMap(s).tobytes() for s in range(n_slots)]
    for f in frames:
        r = W.api.LIB.sdv_lidar_rows_get(W.ctx.p, f, 0, None, C.byref(C.c_int32()), None, None)
        out.append(("rows", f, r, fe.rows(f)["cloud_px"].tobytes() if r == 0 else None))
        cnt = np.zeros(1, np.int32); r = W.api.LIB.sdv_immature_store_count(W.ctx.p, 1, np.array([f], np.uint64), cnt)
        out.append(("store", f, r, S.get(f)[0].tobytes() if r == 0 else None))
    return out


def test_handler_parity(worlds):
    """six sequences of three camera sizes, three consecutive calls (the middle one without stats: it returns at once): after every call each frame's set equals
    the host path (box carried by the host) and the oracle — rows, count, box, flag, numGround, size of segmentedCloud; the slot's box follows the sweep"""
    A, B = worlds; api, synth = A.api, A.synth; n = len(MIX)
    ps = api.PixelSelector(A.ctx, n, A.rp, cams=MIX); fe = api.LidarFrontEnd(A.ctx); feB = api.LidarFrontEnd(B.ctx); of = orc.LidarFrontEnd(); lr = [BOX0] * n
    for call in range(3):
        tlc = synth.TLC if call != 1 else np.array([0.0, -0.08, 0.35]); sw = _sweeps(A, call, upper=(4,)); frames = [fid(j, call) for j in range(n)]
        st = fe.handleRows(list(range(n)), frames, sw, synth.RLC, tlc, _K4(A), stats=(call != 1))
        host = feB.handle(sw, synth.RLC, tlc, _K4(A), lr, cams=MIX)
        for j, c in enumerate(MIX):
            o = of.handle(sw[j], synth.RLC, tlc, A.Ks[c], SIZES[c], lr[j]); g = fe.rows(frames[j])
            for r in (host[j], o):
                assert np.array_equal(g["cloud_px"], r["cloud_px"]) and np.array_equal(g["lrud"], r["lrud"]) and g["addFeaturePoint"] == r["addFeaturePoint"], (call, j)
            assert np.array_equal(ps.lidarBox(j), o["lrud"]) and len(o["cloud_px"]) > 500
            if st is not None:
                assert st[j] == dict(rows=len(o["cloud_px"]), numGround=o["numGround"], n_segmented=o["n_segmented"], addFeaturePoint=o["addFeaturePoint"], overflow=0), (call, j)
                assert (host[j]["numGround"], host[j]["n_segmented"]) == (o["numGround"], o["n_segmented"])
        lr = [r["lrud"] for r in host]
    # the empty sweep, NaN-or-near returns, a sparse sweep: three slots in one call, each starting from the box its slot holds
    full = _sweeps(A, 3)[0]; cases = [np.zeros((0, 4), np.float32), np.array([[np.nan, 0, 0, 0], [0.01, 0.01, 0, 0]], np.float32), full[::7]]; js = [0, 2, 5]
    before = [ps.lidarBox(j).tolist() for j in js]; st = fe.handleRows(js, [9001, 9002, 9003], cases, synth.RLC, synth.TLC, _K4(A, [MIX[j] for j in js]), stats=True)
    for i, j in enumerate(js):
        c = MIX[j]; o = of.handle(cases[i], synth.RLC, synth.TLC, A.Ks[c], SIZES[c], before[i]); g = fe.rows(9001 + i)
        assert np.array_equal(g["cloud_px"], o["cloud_px"]) and np.array_equal(g["lrud"], o["lrud"]) and g["addFeaturePoint"] == o["addFeaturePoint"], i
        assert st[i]["rows"] == len(o["cloud_px"]) and st[i]["n_segmented"] == o["n_segmented"] and st[i]["numGround"] == o["numGround"]
    assert st[0]["rows"] == 0 and st[0]["addFeaturePoint"] == 0 and np.array_equal(ps.lidarBox(0), before[0])
    # the 128-ring sensor
    args = dict(n_scan=128, horizon=1800, ang_res_x=0.2, ang_res_y=0.427 / 2, ang_bottom=24.9, groundScanInd=100)
    wl = synth.World(3000); Rt = synth.trajectory(1, 3000); sw128 = synth.lidar_sweep(wl, Rt[0][0], Rt[1][0], beams=128, seed=3)
    fe128 = api.LidarFrontEnd(A.ctx, **args); b1 = ps.lidarBox(1).tolist(); fe128.handleRows([1], [9004], [sw128], synth.RLC, synth.TLC, _K4(A, [MIX[1]]))
    o = orc.LidarFrontEnd(**args).handle(sw128, synth.RLC, synth.TLC, A.Ks[MIX[1]], SIZES[MIX[1]], b1); g = fe128.rows(9004)
    assert np.array_equal(g["cloud_px"], o["cloud_px"]) and len(o["cloud_px"]) > 6000 and np.array_equal(g["lrud"], o["lrud"]) and np.array_equal(ps.lidarBox(1), o["lrud"])
    fe.dropRows([9001, 9002, 9003, 9004])


def _store(W, frames):
    S = W.api.ImmatureStore(W.ctx); return [b"".join(x.tobytes() for x in S.get(f)) for f in frames]


@pytest.mark.parametrize("async_", [False, True])
def test_make_new_traces_parity(worlds, async_):
    """makeNewTraces from the row sets equals sdv_make_new_traces_store_batch fed the host path's rows, lidar_density of its box and its addFeaturePoint: n_out,
    numPoints, every store block, each slot's potential and selection map; keyframes with addFeaturePoint 1 and 0.  async_: the handler returns at once and
    makeNewTraces follows without a host synchronisation, reading sweeps from pinned host memory that is refilled only after the synchronising call."""
    import torch
    A, B = worlds; api, synth = A.api, A.synth; n = len(MIX); slots = list(range(n))
    psA = api.PixelSelector(A.ctx, n, A.rp, cams=MIX); psB = api.PixelSelector(B.ctx, n, B.rp, cams=MIX); feA = api.LidarFrontEnd(A.ctx); feB = api.LidarFrontEnd(B.ctx)
    lr = [BOX0] * n; flags = set(); pin = torch.empty(0, dtype=torch.float32)
    for k in (0, 1, 2):
        sw = _sweeps(A, k, upper=(1, 4) if k != 1 else (2,)); frames = [fid(j, k) for j in slots]
        if async_:
            sb = np.concatenate([[0], np.cumsum([len(s) for s in sw])]).astype(np.int32)
            if pin.numel() < 4 * int(sb[-1]): pin = torch.empty(4 * int(sb[-1]), dtype=torch.float32).pin_memory()
            buf = pin.numpy()[:4 * int(sb[-1])].reshape(-1, 4); buf[:] = np.concatenate(sw)            # the previous call synchronised: the buffer is free
            assert feA.handleRows(slots, frames, buf, synth.RLC, synth.TLC, _K4(A), sweep_begin=sb) is None
        else:
            feA.handleRows(slots, frames, sw, synth.RLC, synth.TLC, _K4(A), stats=True)
        nA, numA = psA.makeNewTracesRowsStore(slots, frames, DENS, cap=1 << 15)
        host = feB.handle(sw, synth.RLC, synth.TLC, _K4(A), lr, cams=MIX); lr = [r["lrud"] for r in host]
        dl = [api.lidar_density(host[j]["lrud"], SIZES[c], DENS[j]) for j, c in enumerate(MIX)]; add = [r["addFeaturePoint"] for r in host]; flags |= set(add)
        nB, numB = psB.makeNewTracesStore(slots, frames, [r["cloud_px"] for r in host], dl, DENS, add, cap=1 << 15)
        assert np.array_equal(nA, nB) and np.array_equal(numA, numB) and (nA > 100).all(), k
        assert _store(A, frames) == _store(B, frames), k
        for j in slots:
            assert psA.potential(j) == psB.potential(j) and np.array_equal(psA.selectionMap(j), psB.selectionMap(j)) and np.array_equal(psA.lidarBox(j), lr[j]), (k, j)
    assert flags == {0, 1}, flags


def test_keyframe_chain(worlds):
    """sweep -> rows -> makeNewTraces (store) -> traceStoreBatch over the following frames -> activateStoreBatch, against the same chain fed host rows, compared at
    every step; the handler never waits"""
    A, B = worlds; api, synth = A.api, A.synth; n = len(MIX); slots = list(range(n)); hk = [0, 1, 3]
    ps = {W: api.PixelSelector(W.ctx, n, W.rp, cams=MIX) for W in (A, B)}; feA = api.LidarFrontEnd(A.ctx); feB = api.LidarFrontEnd(B.ctx); lr = [BOX0] * n
    for k in hk:
        sw = _sweeps(A, k, upper=(3,)); frames = [fid(j, k) for j in slots]
        feA.handleRows(slots, frames, sw, synth.RLC, synth.TLC, _K4(A)); nA, _ = ps[A].makeNewTracesRowsStore(slots, frames, DENS, cap=1 << 15)
        host = feB.handle(sw, synth.RLC, synth.TLC, _K4(A), lr, cams=MIX); lr = [r["lrud"] for r in host]
        dl = [api.lidar_density(host[j]["lrud"], SIZES[c], DENS[j]) for j, c in enumerate(MIX)]
        nB, _ = ps[B].makeNewTracesStore(slots, frames, [r["cloud_px"] for r in host], dl, DENS, [r["addFeaturePoint"] for r in host], cap=1 << 15)
        assert np.array_equal(nA, nB) and _store(A, frames) == _store(B, frames), k
        if k != 3:
            for kk in (k + 1, k + 2):
                groups = [(j, h) for h in hk if h <= k for j in slots]; geo = [A.geometry(j, h, kk) for j, h in groups]
                cnt = [api.traceStoreBatch(W.ctx, [fid(j, h) for j, h in groups], [fid(j, kk) for j, _ in groups], np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo]),
                                           np.stack([g[2] for g in geo]), cams=[MIX[j] for j, _ in groups], counts=True) for W in (A, B)]
                assert np.array_equal(cnt[0], cnt[1]) and _store(A, [fid(j, h) for j, h in groups]) == _store(B, [fid(j, h) for j, h in groups]), (k, kk)
    seqs = [_window(A, j, hk, 3) for j in slots]
    got = [api.activateStoreBatch(W.ctx, seqs, cams=MIX) for W in (A, B)]
    for key in ("host", "idx", "pts", "meta", "idepth", "res_state", "counts"):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got[0][key], got[1][key])), key
    assert sum(len(x) for x in got[0]["idx"]) > 10
    allf = [fid(j, h) for j in slots for h in hk]
    assert _store(A, allf) == _store(B, allf)
    for W in (A, B):
        api.ImmatureStore(W.ctx).drop(allf)


def test_refusals_overflow_drop_reuse(worlds):
    A, _ = worlds; api, synth = A.api, A.synth; L = api.LIB; cams = [1, 0, 2]
    # no LiDAR front-end / no selector yet: SDV_ERR_STATE
    ctx0 = api.Context(A.Ks[0], *SIZES[0], levels=4, max_frames=4); W0 = type("W0", (), dict(api=api, synth=synth, ctx=ctx0, Ks=A.Ks))()
    sw = _sweeps(A, 0)[:1]
    assert _rows_rc(W0, [0], [1], sw, [0]) == ERR_STATE
    api.LidarFrontEnd(ctx0)
    assert _rows_rc(W0, [0], [1], sw, [0]) == ERR_STATE
    ctx0.close()
    # refusals change no set, box, store block or selector state
    ps = api.PixelSelector(A.ctx, 3, A.rp, cams=cams); fe = api.LidarFrontEnd(A.ctx); S3 = _sweeps(A, 4); F = [fid(j, 4) for j in range(3)]
    fe.handleRows([0, 1, 2], F, S3[:3], synth.RLC, synth.TLC, _K4(A, cams)); ps.makeNewTracesRowsStore([0], [F[0]], 600.0, cap=1 << 15)
    watch = F + [fid(0, 5), 7777]; before = _state(A, ps, fe, 3, watch)
    for slots, frames, cap, want in (([3], [fid(0, 5)], 1 << 15, ERR_ARG), ([0, 0], [fid(0, 5), fid(1, 5)], 1 << 15, ERR_ARG), ([0, 1], [fid(0, 5), fid(0, 5)], 1 << 15, ERR_ARG),
                                     ([0], [fid(0, 5)], 0, ERR_ARG), ([-1], [fid(0, 5)], 1 << 15, ERR_ARG)):
        assert _rows_rc(A, slots, frames, S3[:len(slots)], [cams[max(s, 0) % 3] for s in slots], cap) == want, (slots, frames, cap)
        assert _state(A, ps, fe, 3, watch) == before, (slots, frames, cap)
    nt = lambda s, f: L.sdv_make_new_traces_rows_store_batch(A.ctx.p, 1, np.array([s], np.int32), np.array([f], np.uint64), np.array([600.0], np.float32), 1 << 15,
                                                             np.zeros(1, np.int32), np.zeros(2, np.int32))
    assert nt(1, 7777) == ERR_NOFRAME and nt(1, fid(0, 5)) == ERR_NOFRAME and _state(A, ps, fe, 3, watch) == before
    assert L.sdv_lidar_rows_drop(A.ctx.p, 2, np.array([F[0], 7777], np.uint64)) == ERR_NOFRAME and _state(A, ps, fe, 3, watch) == before
    # overflow: flagged in the stats, refused by get and makeNewTraces (nothing changes); a later deposit with room works
    o = orc.LidarFrontEnd().handle(S3[1], synth.RLC, synth.TLC, A.Ks[cams[1]], SIZES[cams[1]], ps.lidarBox(1).tolist()); nrow = len(o["cloud_px"])
    st = fe.handleRows([1], [F[1]], [S3[1]], synth.RLC, synth.TLC, _K4(A, [cams[1]]), cap=nrow // 2, stats=True)[0]
    assert st == dict(rows=nrow, numGround=o["numGround"], n_segmented=o["n_segmented"], addFeaturePoint=o["addFeaturePoint"], overflow=1)
    no = C.c_int32(0); out = np.zeros((nrow, 3))
    assert L.sdv_lidar_rows_get(A.ctx.p, F[1], nrow, out.ctypes.data, C.byref(no), None, None) == ERR_CAPACITY and no.value == nrow
    mid = _state(A, ps, fe, 3, [F[1]])
    assert nt(1, F[1]) == ERR_CAPACITY and _state(A, ps, fe, 3, [F[1]]) == mid
    box1 = ps.lidarBox(1).tolist(); o = orc.LidarFrontEnd().handle(S3[1], synth.RLC, synth.TLC, A.Ks[cams[1]], SIZES[cams[1]], box1)
    fe.handleRows([1], [F[1]], [S3[1]], synth.RLC, synth.TLC, _K4(A, [cams[1]]), cap=nrow + 10)
    assert np.array_equal(fe.rows(F[1])["cloud_px"], o["cloud_px"]) and nt(1, F[1]) == 0
    # drop, re-deposit, reuse of a handle (a deposit replaces the set), a box set from the host, a rebind to another size restarting the box
    fe.dropRows([F[2]])
    assert L.sdv_lidar_rows_get(A.ctx.p, F[2], 0, None, C.byref(no), None, None) == ERR_NOFRAME and nt(2, F[2]) == ERR_NOFRAME
    for sweep, box in ((S3[2], [300, 900, 60, 200]), (S3[2][::3], None), (S3[0], None)):
        b = ps.lidarBox(2, set_to=box).tolist(); o = orc.LidarFrontEnd().handle(sweep, synth.RLC, synth.TLC, A.Ks[cams[2]], SIZES[cams[2]], b)
        fe.handleRows([2], [F[2]], [sweep], synth.RLC, synth.TLC, _K4(A, [cams[2]]), cap=len(o["cloud_px"]) + 1); g = fe.rows(F[2])
        assert np.array_equal(g["cloud_px"], o["cloud_px"]) and np.array_equal(g["lrud"], o["lrud"]) and np.array_equal(ps.lidarBox(2), o["lrud"])
        assert box is None or b == box
    assert ps.lidarBox(0).tolist() != BOX0
    A.ctx.setCameraSize(3, *SIZES[0]); ps.bindCams([1], [3]); keep = ps.lidarBox(1).tolist()
    assert keep != BOX0
    ps.bindCams([0], [2]); ps.bindCams([1], [2])
    assert ps.lidarBox(0).tolist() == BOX0 and ps.lidarBox(1).tolist() == BOX0 and ps.lidarBox(2).tolist() != BOX0
    fe.dropRows(F); api.ImmatureStore(A.ctx).drop([F[0], F[1]])
