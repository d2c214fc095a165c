"""GPU tests (-m gpu) of the keyframe-rate stages for cameras of different sizes in one context: PixelSelector (makeHists, makeMapsFromLidar, makeMaps),
makeNewTraces, the distance map and activation walk, the LiDAR front-end and the immature-point path (init, traceOn, optimizeImmaturePoint).

The context has KITTI-360's size, 1400x360, on camera 0.  Camera 1 is KITTI (1200x360); camera 2 is 1244x356: w/32 and h/32 leave remainders, level 1 is
622x178 and level 2 is 311 wide.  Every mixed batch interleaves the cameras, and every job must equal, bit for bit, (a) the oracle run at the job's own size
and (b) the same job in a context created at that camera's size."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from test_ref_pin_trace import candidates

pytestmark = pytest.mark.gpu

SIZES = [(1400, 360), (1200, 360), (1244, 356)]
LEVELS = 4
NF = 4                                                     # frames per camera: 0 and 1 are keyframes, 2 and 3 are traced
MIX = [1, 0, 2, 2, 0, 1]                                   # camera of each selector slot / job of a mixed batch
ERR_ARG, ERR_STATE = -1, -5


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def fid(c, k):
    return 100 * c + k


class World:
    """the three cameras' sequences, the mixed context and one context per camera size holding the same frames"""

    def __init__(self):
        api, synth = _mods(); self.api, self.synth = api, synth
        self.Ks = [tuple(synth.K360_K), tuple(synth.KITTI_K), (702.5, 698.0, 611.0, 171.5)]
        self.seqs = [cached_sequence(NF, 5100 + c, self.Ks[c], SIZES[c]) for c in range(3)]
        self.of = [[orc.Frame(im, LEVELS) for im in s.images] for s in self.seqs]
        self.rps = [api.random_pattern(*wh) for wh in SIZES]
        self.poses = [[np.concatenate([synth._quat_from_R(s.R[i]), s.t[i]]) for i in range(NF)] for s in self.seqs]
        self.ctx = api.Context(self.Ks[0], *SIZES[0], levels=LEVELS, max_frames=32, max_kf_images=32)
        for c in (1, 2):
            self.ctx.setCameraSize(c, *SIZES[c])
        self.singles = [api.Context(self.Ks[c], *SIZES[c], levels=LEVELS, max_frames=16, max_kf_images=16) for c in range(3)]
        for c in range(3):
            ims = [np.ascontiguousarray(im, np.float32) for im in self.seqs[c].images]; ids = [fid(c, k) for k in range(NF)]
            self.ctx.makeImagesBatch(ids, [a.ctypes.data for a in ims], cams=[c] * NF); self.ctx.sync()
            self.singles[c].makeImagesBatch(ids, [a.ctypes.data for a in ims]); self.singles[c].sync()

    def single_selector(self, c, n):
        return self.api.PixelSelector(self.singles[c], n, self.rps[c])


@pytest.fixture(scope="module")
def world():
    w = World()
    yield w
    w.ctx.close()
    for s in w.singles:
        s.close()


def _jobs_of(c):
    return [j for j, cc in enumerate(MIX) if cc == c]


def test_hists_and_make_maps_mixed(world):
    W = world; api = W.api; n = len(MIX)
    ps = api.PixelSelector(W.ctx, n, W.rps[0], cams=MIX)
    for c in (2, 0, 1):
        a, b = ps.makeHists(fid(c, 1), cam=c); oa, ob = orc.Selector(*SIZES[c], W.rps[c]).makeHists(W.of[c][1]); sa, sb = W.single_selector(c, 1).makeHists(fid(c, 1))
        assert len(a) == (SIZES[c][0] // 32) * (SIZES[c][1] // 32) and np.array_equal(a, oa) and np.array_equal(b, ob) and np.array_equal(a, sa) and np.array_equal(b, sb), c
    sps = [W.single_selector(c, n) for c in range(3)]
    for pots, dens, recs, ths in (([3, 2, 4, 5, 2, 3], [500., 1500., 60., 2500., 900., 333.], [1, 1, 1, 1, 0, 1], [1.0, 1.0, 1.0, 2.0, 1.0, 1.0]),
                                  ([1, 8, 3, 2, 6, 4], [3000., 100., 1e5, 700., 1200., 50.], [1, 1, 0, 1, 1, 1], [1.0, 1.5, 1.0, 1.0, 1.0, 1.0])):
        for lidar in (True, False):
            frames = [fid(c, j % 2) for j, c in enumerate(MIX)]; clouds = [W.seqs[c].clouds[j % 2] for j, c in enumerate(MIX)] if lidar else None
            for j in range(n): ps.potential(j, pots[j])
            maps, num = ps.makeMapsBatch(list(range(n)), frames, dens, recs, ths, clouds)
            assert isinstance(maps, list)
            for c in range(3):
                js = _jobs_of(c)
                for j in js: sps[c].potential(j, pots[j])
                smaps, snum = sps[c].makeMapsBatch(js, [frames[j] for j in js], [dens[j] for j in js], [recs[j] for j in js], [ths[j] for j in js], [clouds[j] for j in js] if lidar else None)
                for i, j in enumerate(js):
                    o = orc.Selector(*SIZES[c], W.rps[c]); o.currentPotential = pots[j]
                    m, nh = o.makeMaps(W.of[c][j % 2], dens[j], recs[j], ths[j], clouds[j] if lidar else None)
                    assert nh == num[j] == snum[i] and o.currentPotential == ps.potential(j) == sps[c].potential(j), (lidar, j, c)
                    assert np.array_equal(m.astype(np.uint8), maps[j]) and np.array_equal(maps[j], smaps[i]), (lidar, j, c)
                    if not lidar:
                        assert maps[j].shape == SIZES[c][::-1] and np.array_equal(ps.selectionMap(j), maps[j])


@pytest.mark.parametrize("add_feature", [0, 1])
def test_make_new_traces_mixed(world, add_feature):
    """two keyframe rounds on slots of three sizes: records, ImmaturePoint bytes, numPoints, potentials, selection maps at each slot's size"""
    W = world; api = W.api; n = len(MIX); dens = [600.0, 1500.0, 300.0, 900.0, 450.0, 1200.0]
    ps = api.PixelSelector(W.ctx, n, W.rps[0], cams=MIX); sps = [W.single_selector(c, n) for c in range(3)]
    osel = [orc.Selector(*SIZES[c], W.rps[c]) for c in MIX]; omap = [np.zeros(SIZES[c][::-1], np.float32) for c in MIX]
    for rnd in range(2):
        fr = [(j + rnd) % 2 for j in range(n)]; clouds = [W.seqs[c].clouds[fr[j]] for j, c in enumerate(MIX)]
        lr = [[int(c[:, 0].min()), int(c[:, 0].max()), int(c[:, 1].min()), int(c[:, 1].max())] for c in clouds]
        dl = [api.lidar_density(lr[j], SIZES[c], dens[j]) for j, c in enumerate(MIX)]; add = [int(add_feature and not (rnd == 1 and j == 1)) for j in range(n)]
        res, num = ps.makeNewTracesBatch(list(range(n)), [fid(c, fr[j]) for j, c in enumerate(MIX)], clouds, dl, dens, add, cap=1 << 15)
        for c in range(3):
            js = _jobs_of(c)
            sres, snum = sps[c].makeNewTracesBatch(js, [fid(c, fr[j]) for j in js], [clouds[j] for j in js], [dl[j] for j in js], [dens[j] for j in js], [add[j] for j in js], cap=1 << 15)
            for i, j in enumerate(js):
                T, onum, _ = osel[j].makeNewTraces(W.of[c][fr[j]], clouds[j], dl[j], dens[j], add[j], omap[j]); G, I = res[j]
                assert T.tobytes() == G.tobytes() == sres[i][0].tobytes() and np.array_equal(onum, num[j]) and np.array_equal(num[j], snum[i]), (rnd, j, c)
                assert osel[j].currentPotential == ps.potential(j) == sps[c].potential(j)
                assert np.array_equal(omap[j].astype(np.uint8), ps.selectionMap(j)) and np.array_equal(ps.selectionMap(j), sps[c].selectionMap(j))
                P = orc.immature_init(W.of[c][fr[j]], np.stack([T["u"], T["v"]], 1).astype(np.int32))
                assert P.tobytes() == I.tobytes() == sres[i][1].tobytes(), (rnd, j, c)
                assert len(T) > 100 and (T["type"] == 0).sum() > 0


def _act_inputs(W, c, rng, minActDist):
    """sources: cloud pixels of keyframes 0, 1 of camera c's sequence; candidates of keyframes 0, 1, 2 (random pixels, some projecting outside); newest = frame 3"""
    synth = W.synth; K = W.Ks[c]; seq = W.seqs[c]; w, h = SIZES[c]; K0, K1 = orc.distmap_geometry(K, None, None); Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
    def geo(hh):
        R, t = synth.rel_pose(seq.R[hh], seq.t[hh], seq.R[3], seq.t[3]); return (K1 @ R.astype(np.float32) @ Ki0).astype(np.float32), (K1 @ t.astype(np.float32)).astype(np.float32)
    G = [geo(hh) for hh in (0, 1, 2)]; uvid, pb = [], [0]
    for hh in (0, 1):
        cl = seq.clouds[hh]; pick = rng.choice(len(cl), 150, replace=False); uvid.append(np.stack([np.floor(cl[pick, 0]), np.floor(cl[pick, 1]), 1.0 / cl[pick, 2]], 1)); pb.append(pb[-1] + 150)
    cb = [0]; cand = []
    for nn in (400, 300, 150):
        u = rng.integers(4, w - 5, nn); v = rng.integers(4, h - 5, nn); idm = rng.uniform(0.01, 0.4, nn).astype(np.float32); idm[:6] = 6.0
        cand.append(np.stack([u, v, idm, rng.choice([1.0, 2.0, 4.0], nn)], 1).astype(np.float32)); cb.append(cb[-1] + nn)
    return dict(pt_begin=np.array(pb, np.int32), KRKi=np.stack([G[0][0], G[1][0]]), Kt=np.stack([G[0][1], G[1][1]]), uvid=np.concatenate(uvid).astype(np.float32),
                cand_begin=np.array(cb, np.int32), cKRKi=np.stack([g[0] for g in G]), cKt=np.stack([g[1] for g in G]), cand4=np.concatenate(cand), minActDist=minActDist)


def test_activation_mixed(world):
    W = world; api = W.api; rng = np.random.default_rng(11)
    api.PixelSelector(W.ctx, 1, W.rps[0]); sps = [W.single_selector(c, 1) for c in range(3)]
    seqs = [_act_inputs(W, c, rng, d) for c, d in zip(MIX, (0.0, 1.0, 2.5, 1.5, 4.0, 2.0))]
    decs, maps = api.activateSelectBatch(W.ctx, seqs, want_maps=True, cams=MIX)
    for c in range(3):
        js = _jobs_of(c); sdec, smaps = api.activateSelectBatch(W.singles[c], [seqs[j] for j in js], want_maps=True)
        for i, j in enumerate(js):
            q = seqs[j]; od = orc.DistMap(SIZES[c][0] >> 1, SIZES[c][1] >> 1); od.make(q["pt_begin"], q["KRKi"], q["Kt"], q["uvid"])
            do = od.activateSelect(q["cand_begin"], q["cKRKi"], q["cKt"], q["cand4"], q["minActDist"])
            assert maps[j].shape == (SIZES[c][1] >> 1, SIZES[c][0] >> 1) and np.array_equal(maps[j], od.get()) and np.array_equal(maps[j], smaps[i]), (j, c)
            assert np.array_equal(decs[j], do) and np.array_equal(decs[j], sdec[i]), (j, c)
            assert (do == 1).sum() > 10 and (do == -1).sum() >= 1


def test_lidar_front_end_mixed(world):
    """raw sweeps of three cameras in one call, pixel box carried over a second call: each camera's size bounds its box and its border test"""
    W = world; api, synth = W.api, W.synth
    world_ = synth.World(5100); R, t = synth.trajectory(3, 5100)
    S = [synth.lidar_sweep(world_, R[j % 3], t[j % 3], seed=j) for j in range(len(MIX))]; K4 = np.array([W.Ks[c] for c in MIX], np.float32)
    G = api.LidarFrontEnd(W.ctx); singles = [api.LidarFrontEnd(W.singles[c]) for c in range(3)]; fe = orc.LidarFrontEnd(); lr0 = [[10000, -1, 10000, -1]] * len(MIX)
    for rnd in range(2):
        tlc = synth.TLC if rnd == 0 else np.array([0.0, -0.08, 0.35])
        res = G.handle(S, synth.RLC, tlc, K4, lr0, cams=MIX)
        for c in range(3):
            js = _jobs_of(c); sres = singles[c].handle([S[j] for j in js], synth.RLC, tlc, W.Ks[c], [lr0[j] for j in js])
            for i, j in enumerate(js):
                o = fe.handle(S[j], synth.RLC, tlc, W.Ks[c], SIZES[c], lr0[j])
                for r in (res[j], sres[i]):
                    assert np.array_equal(o["cloud_px"], r["cloud_px"]) and np.array_equal(o["lrud"], r["lrud"]), (rnd, j, c)
                    assert (o["numGround"], o["n_segmented"], o["addFeaturePoint"]) == (r["numGround"], r["n_segmented"], r["addFeaturePoint"])
                assert len(o["cloud_px"]) > 3000 and o["cloud_px"][:, 0].max() < SIZES[c][0] - 5
        lr0 = [r["lrud"] for r in res]


def _pre14(synth, seq, host, tgt):
    R, t = synth.rel_pose(seq.R[host], seq.t[host], seq.R[tgt], seq.t[tgt])
    return np.concatenate([np.asarray(R, np.float32).reshape(-1), np.asarray(t, np.float32), [1.0, 0.0]]).astype(np.float32)


def test_immature_points_mixed(world):
    """ImmaturePoint ctor per camera, traceOn of groups of three cameras in one launch over two traced frames, optimizeImmaturePoint of groups of three cameras"""
    W = world; api, synth = W.api, W.synth; groups = [(c, host) for host in (0, 1) for c in (1, 0, 2)]
    P, Po, Ps = [], [], []
    for c, host in groups:
        uv = candidates(W.seqs[c], 500, 40 + 10 * c + host); uv[:6] = np.clip(uv[:6], 3, [SIZES[c][0] - 4, SIZES[c][1] - 4])
        p = api.immatureInit(W.ctx, fid(c, host), uv, cam=c); po = orc.immature_init(W.of[c][host], uv); pss = api.immatureInit(W.singles[c], fid(c, host), uv)
        assert p.tobytes() == po.tobytes() == pss.tobytes(), (c, host)
        P.append(p); Po.append(po); Ps.append(pss)
    pb = np.cumsum([0] + [len(p) for p in P]).astype(np.int32); cams = [c for c, _ in groups]; allp = np.concatenate(P); seen = set()
    for k, (ab, ex) in zip((2, 3), (((0.0, 0.0), 1.0), ((0.02, -1.5), 1.1))):
        geo = [orc.trace_geometry(W.Ks[c], W.poses[c][host], W.poses[c][k], 1.0, ex, (0.0, 0.0), ab) for c, host in groups]
        st = api.traceOnBatch(W.ctx, [fid(c, k) for c in cams], pb, np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo]), np.stack([g[2] for g in geo]), allp, cams=cams)
        for g, (c, host) in enumerate(groups):
            so = orc.immature_trace(W.of[c][k], Po[g], *geo[g]); ss = api.traceOnBatch(W.singles[c], [fid(c, k)], [0, len(Ps[g])], geo[g][0][None], geo[g][1][None], geo[g][2][None], Ps[g])
            assert np.array_equal(st[pb[g]:pb[g + 1]], so) and np.array_equal(so, ss), (k, c, host)
            assert allp[pb[g]:pb[g + 1]].tobytes() == Po[g].tobytes() == Ps[g].tobytes(), (k, c, host)
            seen |= set(so.tolist())
    assert {api.IPS_GOOD, api.IPS_OOB} <= seen, seen
    # optimizeImmaturePoint: host 0 of each camera against targets 1..3, interleaved
    og = [1, 0, 2]; rng = np.random.default_rng(7); gp, want, sgot = [], [], []
    for c in og:
        p = Po[groups.index((c, 0))].copy(); bad = ~np.isfinite(p["idepth_max"]); p["idepth_max"][bad] = 0.2; p["idepth_min"][bad] = 0.0
        sensor = rng.uniform(size=len(p)) < 0.15; pre = np.stack([_pre14(synth, W.seqs[c], 0, t) for t in (1, 2, 3)]); K = W.Ks[c]
        cal = np.array([K[0], K[1], K[2], K[3], 1.0 / K[0], 1.0 / K[1]], np.float32)
        want.append(orc.immature_optimize(p, sensor, [W.of[c][t] for t in (1, 2, 3)], pre, cal, 1))
        sgot.append(api.optimizeImmaturePointBatch(W.singles[c], [0, len(p)], [0, 3], [fid(c, t) for t in (1, 2, 3)], pre, cal[None], p.view(api.IMMATURE_PT_DTYPE), sensor, 1))
        gp.append((p, sensor, pre, cal))
    pts = np.concatenate([g[0] for g in gp]).view(api.IMMATURE_PT_DTYPE); opb = np.cumsum([0] + [len(g[0]) for g in gp]); tb = [0, 3, 6, 9]
    st, idp, rs = api.optimizeImmaturePointBatch(W.ctx, opb, tb, [fid(c, t) for c in og for t in (1, 2, 3)], np.concatenate([g[2] for g in gp]), np.stack([g[3] for g in gp]), pts,
                                                 np.concatenate([g[1] for g in gp]), 1, cams=og)
    for g, c in enumerate(og):
        so, io, ro = want[g]; a = slice(opb[g], opb[g + 1]); act = so == 1
        assert np.array_equal(st[a], so) and np.array_equal(so, sgot[g][0]), c
        assert np.array_equal(idp[a][act], io[act]) and np.array_equal(rs[a][act], ro[act]) and np.array_equal(idp[a], sgot[g][1]) and np.array_equal(rs[a], sgot[g][2]), c
        assert act.sum() > 20, c


def test_refusals_change_nothing(world):
    W = world; api, synth = W.api, W.synth; L = api.LIB; ctx = W.ctx
    ps = api.PixelSelector(ctx, 3, W.rps[0], cams=[1, 0, 2]); cl = W.seqs[1].clouds[0]
    ps.makeNewTracesBatch([0], [fid(1, 0)], [cl], 300.0, 600.0, 1); pot0, map0 = ps.potential(0), ps.selectionMap(0)
    assert map0.shape == (360, 1200) and map0.any()
    # a frame of another size on a bound slot: refused, nothing changed
    for call in (lambda: ps.makeNewTracesBatch([0], [fid(0, 0)], [cl], 300.0, 600.0, 1), lambda: ps.makeMapsBatch([0], [fid(2, 0)], 500.0),
                 lambda: ps.makeMapsBatch([1, 0], [fid(0, 0), fid(0, 1)], 500.0, clouds=[cl, cl])):
        with pytest.raises(api.SdvError):
            call()
        assert ps.potential(0) == pot0 and np.array_equal(ps.selectionMap(0), map0)
    # a camera out of range
    for call in (lambda: ps.bindCams([0], [8]), lambda: ps.bindCams([5], [1]), lambda: ps.makeHists(fid(1, 0), cam=-1),
                 lambda: api.immatureInit(ctx, fid(1, 0), [[50, 50]], cam=9), lambda: api.activateSelectBatch(ctx, [dict(pt_begin=[0], KRKi=np.zeros((0, 9)), Kt=np.zeros((0, 3)), uvid=np.zeros((0, 3)))], cams=[8])):
        with pytest.raises(api.SdvError):
            call()
    assert ps.potential(0) == pot0 and np.array_equal(ps.selectionMap(0), map0) and ps.slotSize(0) == SIZES[1]
    # rebinding: a camera of the same size keeps the slot's state, another size starts it afresh
    ctx.setCameraSize(3, *SIZES[1]); ps.bindCams([0], [3])
    assert ps.potential(0) == pot0 and np.array_equal(ps.selectionMap(0), map0)
    ps.bindCams([0], [2])
    assert ps.potential(0) == 3 and ps.selectionMap(0).shape == (356, 1244) and not ps.selectionMap(0).any()
    # sdv_set_camera_size on a camera with bound selector slots
    ctx.setCameraSize(4, 1200, 352); ps.bindCams([2], [4])
    assert L.sdv_set_camera_size(ctx.p, 4, 1000, 300) == ERR_STATE
    ps.bindCams([2], [0]); ctx.setCameraSize(4, 1000, 300)
    # the camera-less entries still mean camera 0 and refuse camera-1 frames
    uv = np.array([[50, 50], [100, 80]], np.int32)
    with pytest.raises(api.SdvError):
        api.immatureInit(ctx, fid(1, 0), uv)
    P = api.immatureInit(ctx, fid(1, 0), uv, cam=1); Pb = P.copy(); I3 = np.eye(3, dtype=np.float32)[None]; z3 = np.zeros((1, 3), np.float32); a2 = np.array([[1, 0]], np.float32)
    for call in (lambda: api.traceOnBatch(ctx, [fid(1, 2)], [0, 2], I3, z3, a2, P), lambda: api.traceOnBatch(ctx, [fid(0, 2)], [0, 2], I3, z3, a2, P, cams=[1]),
                 lambda: ps.makeHists(fid(1, 0))):
        with pytest.raises(api.SdvError):
            call()
    assert P.tobytes() == Pb.tobytes()
    ctx.setCameraSize(3, *SIZES[0])


def test_end_to_end_kitti360_and_kitti_in_one_context(world):
    """KITTI-360 and KITTI drives interleaved in every batch, one keyframe step each: LiDAR handler -> makeNewTraces -> traceOn into the next frames ->
    activation.  Everything equals two contexts of one size each, bit for bit."""
    W = world; api, synth = W.api, W.synth; cams = [0, 1, 0, 1]; n = len(cams)
    world_ = synth.World(5200); R, t = synth.trajectory(2, 5200); S = [synth.lidar_sweep(world_, R[j % 2], t[j % 2], seed=10 + j) for j in range(n)]
    def run(ctx, js, cam_arg):
        """the keyframe step of sequences js (all in ctx) -> everything it produced"""
        m = len(js); cm = [cams[j] for j in js] if cam_arg else None; out = {}
        fe = api.LidarFrontEnd(ctx); K4 = np.array([W.Ks[cams[j]] for j in js], np.float32)
        lid = fe.handle([S[j] for j in js], synth.RLC, synth.TLC, K4, [[10000, -1, 10000, -1]] * m, cams=cm)
        ps = api.PixelSelector(ctx, m, W.rps[0] if cam_arg else W.rps[cams[js[0]]], cams=cm)
        dl = [api.lidar_density(lid[i]["lrud"], SIZES[cams[j]], 1500.0) for i, j in enumerate(js)]
        res, num = ps.makeNewTracesBatch(list(range(m)), [fid(cams[j], 0) for j in js], [r["cloud_px"] for r in lid], dl, 1500.0, [r["addFeaturePoint"] for r in lid], cap=1 << 15)
        pts = np.concatenate([r[1] for r in res]).copy(); pb = np.cumsum([0] + [len(r[1]) for r in res]).astype(np.int32)
        sts = []
        for k in (1, 2):
            geo = [orc.trace_geometry(W.Ks[cams[j]], W.poses[cams[j]][0], W.poses[cams[j]][k]) for j in js]
            sts.append(api.traceOnBatch(ctx, [fid(cams[j], k) for j in js], pb, np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo]), np.stack([g[2] for g in geo]), pts, cams=cm))
        seqs = []
        for i, j in enumerate(js):
            c = cams[j]; p = pts[pb[i]:pb[i + 1]]; good = p["lastTraceStatus"] == api.IPS_GOOD
            K0, K1 = orc.distmap_geometry(W.Ks[c], None, None); Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
            Rr, tr = synth.rel_pose(W.seqs[c].R[0], W.seqs[c].t[0], W.seqs[c].R[3], W.seqs[c].t[3]); A = (K1 @ Rr.astype(np.float32) @ Ki0).astype(np.float32); B = (K1 @ tr.astype(np.float32)).astype(np.float32)
            cl = lid[i]["cloud_px"][::5]; uvid = np.stack([np.floor(cl[:, 0]), np.floor(cl[:, 1]), 1.0 / cl[:, 2]], 1).astype(np.float32)
            cand4 = np.stack([p["u"][good], p["v"][good], 0.5 * (p["idepth_max"][good] + p["idepth_min"][good]), res[i][0]["my_type"][good]], 1).astype(np.float32)
            seqs.append(dict(pt_begin=[0, len(uvid)], KRKi=A[None], Kt=B[None], uvid=uvid, cand_begin=[0, len(cand4)], cKRKi=A[None], cKt=B[None], cand4=cand4, minActDist=2.0))
        decs, maps = api.activateSelectBatch(ctx, seqs, want_maps=True, cams=cm)
        for i, j in enumerate(js):
            out[j] = dict(lid=lid[i], rec=res[i][0].tobytes(), num=num[i].tolist(), pts=pts[pb[i]:pb[i + 1]].tobytes(), st=[s[pb[i]:pb[i + 1]].tolist() for s in sts],
                          map=ps.selectionMap(i), dec=decs[i].tolist(), dmap=maps[i], pot=ps.potential(i))
        return out
    mixed = run(W.ctx, list(range(n)), True); ref = {}
    for c in (0, 1):
        ref.update(run(W.singles[c], [j for j in range(n) if cams[j] == c], False))
    for j in range(n):
        a, b = mixed[j], ref[j]
        assert np.array_equal(a["lid"]["cloud_px"], b["lid"]["cloud_px"]) and np.array_equal(a["lid"]["lrud"], b["lid"]["lrud"]) and a["lid"]["addFeaturePoint"] == b["lid"]["addFeaturePoint"], j
        assert a["rec"] == b["rec"] and a["num"] == b["num"] and a["pts"] == b["pts"] and a["st"] == b["st"] and a["pot"] == b["pot"], j
        assert np.array_equal(a["map"], b["map"]) and a["dec"] == b["dec"] and np.array_equal(a["dmap"], b["dmap"]), j
        assert len(a["rec"]) > 100 * 28 and 1 in a["dec"] and a["map"].shape == SIZES[cams[j]][::-1]
