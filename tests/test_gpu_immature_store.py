"""GPU tests (-m gpu) of the device-resident immature-point store: host->immaturePoints of every keyframe kept on the device, filled by makeNewTraces, traced by
traceNewCoarse every frame, dropped with the keyframe.  Every result is compared bit for bit with the host-record entries the store replaces
(sdv_make_new_traces_batch + the host-side rules of FullSystem.cpp:1313-1317 and :1080-1084, sdv_immature_trace_batch_cams), and the store's trace with the
reference's own traceNewCoarse (tests/golden/seq_trace_ref.npz).

The mixed context has KITTI-360's size, 1400x360, on camera 0, KITTI (1200x360) on camera 1 and 1244x356 on camera 2; every batch interleaves the cameras."""
import ctypes
import os
import numpy as np
import pytest
import orc
from conftest import cached_sequence
from ref_golden import _digest

pytestmark = pytest.mark.gpu

SIZES = [(1400, 360), (1200, 360), (1244, 356)]
LEVELS = 4
NF = 6                                                     # frames per sequence
MIX = [1, 0, 2, 2, 0, 1]                                   # camera of each sequence (= selector slot) of the batch
DENS = [600.0, 1500.0, 300.0, 900.0, 450.0, 1200.0]
ERR_ARG, ERR_NOFRAME, ERR_CAPACITY = -1, -3, -4
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seq_trace_ref.npz")


def _mods():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api, synth
    return api, synth


def fid(j, k):
    return 100 * j + k


class World:
    """one sequence per entry of MIX (the sequences of one camera share its synthetic drive, under their own frame ids) in one mixed context"""

    def __init__(self):
        api, synth = _mods(); self.api, self.synth = api, synth
        self.Ks = [tuple(synth.K360_K), tuple(synth.KITTI_K), (702.5, 698.0, 611.0, 171.5)]
        self.seqs = [cached_sequence(NF, 5300 + c, self.Ks[c], SIZES[c]) for c in range(3)]
        self.poses = [[np.concatenate([synth._quat_from_R(s.R[i]), s.t[i]]) for i in range(NF)] for s in self.seqs]
        self.rp = api.random_pattern(*SIZES[0])
        self.ctx = api.Context(self.Ks[0], *SIZES[0], levels=LEVELS, max_frames=64, max_kf_images=64)
        for c in (1, 2):
            self.ctx.setCameraSize(c, *SIZES[c])
        for j, c in enumerate(MIX):
            ims = [np.ascontiguousarray(im, np.float32) for im in self.seqs[c].images]
            self.ctx.makeImagesBatch([fid(j, k) for k in range(NF)], [a.ctypes.data for a in ims], cams=[c] * NF); self.ctx.sync()

    def clouds(self, k):
        return [self.seqs[c].clouds[k] for c in MIX]

    def densities(self, k):
        lr = [[int(cl[:, 0].min()), int(cl[:, 0].max()), int(cl[:, 1].min()), int(cl[:, 1].max())] for cl in self.clouds(k)]
        return [self.api.lidar_density(lr[j], SIZES[c], DENS[j]) for j, c in enumerate(MIX)]

    def geometry(self, j, host_k, new_k):
        c = MIX[j]; ab = ((0.0, 0.0), (0.01 * new_k, -0.5 * new_k)); ex = (1.0, 1.0 + 0.02 * (new_k - host_k))
        return orc.trace_geometry(self.Ks[c], self.poses[c][host_k], self.poses[c][new_k], ex[0], ex[1], ab[0], ab[1])


@pytest.fixture(scope="module")
def world():
    w = World()
    yield w
    w.ctx.close()


def _after_make_key_frame(api, T, I):
    """what the reference's ImmaturePoints hold after makeNewTraces (:1313-1317) and makeKeyFrame's loop (:1080-1084), as records + meta"""
    P = I.copy(); s = T["isFromSensor"] != 0
    P["idepth_min"][s] = T["idepth_fromSensor"][s]; P["idepth_max"][s] = T["idepth_fromSensor"][s]; P["lastTraceStatus"][s] = api.IPS_SKIPPED
    M = np.zeros(len(T), api.IMMATURE_META_DTYPE)
    for f in ("my_type", "type", "isFromSensor", "idepth_fromSensor"):
        M[f] = T[f]
    return P, M


def _hist(st):
    return np.bincount(np.asarray(st, np.int64), minlength=6)[:6]


def test_store_round_trip_and_refusals(world):
    W = world; api = W.api; L = api.LIB; ctx = W.ctx; S = api.ImmatureStore(ctx); rng = np.random.default_rng(3)
    P = api.immatureInit(ctx, fid(0, 0), np.stack([rng.integers(8, 1100, 700), rng.integers(8, 340, 700)], 1), cam=1)
    P["lastTraceStatus"] = rng.integers(0, 6, len(P)); P["quality"] = rng.uniform(0, 10, len(P)).astype(np.float32)
    M = np.zeros(len(P), api.IMMATURE_META_DTYPE); M["my_type"] = rng.choice([1.0, 2.0, 4.0], len(P)); M["type"] = rng.integers(-1, 2, len(P)); M["isFromSensor"] = M["type"] >= 0
    M["idepth_fromSensor"] = rng.uniform(0.01, 0.5, len(P))
    S.set(7001, P, M); S.set(7002, P[:300]); S.set(7003, P[:0])
    assert S.count([7001, 7002, 7003]).tolist() == [700, 300, 0]
    g, m = S.get(7001); assert g.tobytes() == P.tobytes() and m.tobytes() == M.tobytes()
    g, m = S.get(7002); assert g.tobytes() == P[:300].tobytes() and np.all(m["my_type"] == 1) and np.all(m["type"] == -1) and not m["isFromSensor"].any()
    S.set(7002, P[::-1].copy(), M[::-1].copy()); g, m = S.get(7002)                      # a larger replacement moves the host to a bigger block
    assert g.tobytes() == P[::-1].tobytes() and m.tobytes() == M[::-1].tobytes()
    S.set(7001, P[:10], M[:10]); g, _ = S.get(7001); assert g.tobytes() == P[:10].tobytes()   # a smaller one stays in place
    # refusals change nothing
    cnt = ctypes.c_int32(0); buf = np.zeros(5, api.IMMATURE_PT_DTYPE)
    assert L.sdv_immature_store_get(ctx.p, 7002, 5, buf.ctypes.data, None, ctypes.byref(cnt)) == ERR_CAPACITY and cnt.value == 700 and not buf.view(np.uint8).any()
    assert L.sdv_immature_store_get(ctx.p, 9999, 5, buf.ctypes.data, None, ctypes.byref(cnt)) == ERR_NOFRAME
    assert L.sdv_immature_store_count(ctx.p, 2, np.array([7001, 9999], np.uint64), np.zeros(2, np.int32)) == ERR_NOFRAME
    assert L.sdv_immature_store_drop(ctx.p, 2, np.array([7001, 9999], np.uint64)) == ERR_NOFRAME
    I3 = np.eye(3, dtype=np.float32).reshape(-1); z3 = np.zeros(3, np.float32); a2 = np.array([1, 0], np.float32)
    tr = lambda hosts, frames, cams: L.sdv_immature_trace_store_batch(ctx.p, len(hosts), np.array(hosts, np.uint64), np.array(frames, np.uint64),
                                                                       None if cams is None else np.array(cams, np.int32).ctypes.data, np.tile(I3, len(hosts)),
                                                                       np.tile(z3, len(hosts)), np.tile(a2, len(hosts)), None)
    assert tr([9999], [fid(0, 1)], [1]) == ERR_NOFRAME                                    # unknown host
    assert tr([7002], [55555], [1]) == ERR_NOFRAME                                         # unknown traced frame
    assert tr([7002], [fid(0, 1)], [8]) == ERR_ARG and tr([7002], [fid(0, 1)], [-1]) == ERR_ARG   # camera out of range
    assert tr([7002], [fid(0, 1)], None) == ERR_ARG                                        # a camera-1 frame traced at camera 0's size
    assert tr([7002, 7002], [fid(0, 1), fid(0, 2)], [1, 1]) == ERR_ARG                     # one host twice
    assert L.sdv_immature_store_set(ctx.p, 7005, -1, None, None) == ERR_ARG
    assert S.count([7001, 7002, 7003]).tolist() == [10, 700, 0]
    g, m = S.get(7002); assert g.tobytes() == P[::-1].tobytes() and m.tobytes() == M[::-1].tobytes()
    with pytest.raises(api.SdvError):
        api.traceStoreBatch(ctx, [7002], [fid(0, 1)], I3[None], z3[None], a2[None], cams=[0])
    S.drop([7001, 7002, 7003])
    for h in (7001, 7002, 7003):
        with pytest.raises(api.SdvError):
            S.count([h])
    S.set(7004, P); g, _ = S.get(7004); assert g.tobytes() == P.tobytes()                  # a dropped block is reused
    S.drop(7004)


@pytest.mark.parametrize("add_feature", [0, 1])
def test_deposit_equals_make_new_traces(world, add_feature):
    """two keyframe rounds: the store's blocks equal sdv_make_new_traces_batch's records after the host-side rules, for slots of three sizes"""
    W = world; api = W.api; n = len(MIX); S = api.ImmatureStore(W.ctx)
    ps = api.PixelSelector(W.ctx, 2 * n, W.rp, cams=MIX + MIX)                           # slots 0..n-1: host records, n..2n-1: the store
    for rnd, k in enumerate((0, 1)):
        add = [int(add_feature and not (rnd == 1 and j == 1)) for j in range(n)]; frames = [fid(j, k) for j in range(n)]
        res, num = ps.makeNewTracesBatch(list(range(n)), frames, W.clouds(k), W.densities(k), DENS, add, cap=1 << 15)
        n_out, num_s = ps.makeNewTracesStore(list(range(n, 2 * n)), frames, W.clouds(k), W.densities(k), DENS, add, cap=1 << 15)
        assert np.array_equal(num, num_s) and S.count(frames).tolist() == n_out.tolist() == [len(r[0]) for r in res]
        for j in range(n):
            P, M = _after_make_key_frame(api, *res[j]); g, m = S.get(frames[j])
            assert g.tobytes() == P.tobytes() and m.tobytes() == M.tobytes(), (rnd, j)
            assert ps.potential(j) == ps.potential(n + j) and np.array_equal(ps.selectionMap(j), ps.selectionMap(n + j))
            assert len(P) > 100 and (M["isFromSensor"] == 1).any() and (P["lastTraceStatus"] == api.IPS_SKIPPED).any()
            if add[j]:
                assert (M["type"] == -1).any()
    S.drop([fid(j, k) for j in range(n) for k in (0, 1)])


def test_drive_deposit_trace_drop(world):
    """a drive of six mixed sequences over NF frames: keyframes 0, 1 and 3 deposit their candidates; every frame traces the window's keyframes into it; keyframe 0
    leaves the window before frame 5.  The store carries the state on the device only; after every step each block equals the host-record loop
    (sdv_make_new_traces_batch + host rules, sdv_immature_trace_batch_cams on one host array), and counts_out equals the status histogram."""
    W = world; api = W.api; n = len(MIX); S = api.ImmatureStore(W.ctx)
    ps = api.PixelSelector(W.ctx, 2 * n, W.rp, cams=MIX + MIX)
    host = {}                                                                              # (j, keyframe) -> records of the host-record path
    window = []; seen = set()
    for k in range(NF):
        if window:
            if k == 5:
                S.drop([fid(j, 0) for j in range(n)]); window.remove(0)
                for j in range(n):
                    del host[(j, 0)]
            groups = [(j, h) for h in window for j in range(n)]                          # host-major, sequences interleaved: three cameras in one launch
            geo = [W.geometry(j, h, k) for j, h in groups]
            KR, Kt, aff = np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo]), np.stack([g[2] for g in geo])
            cams = [MIX[j] for j, _ in groups]
            counts = api.traceStoreBatch(W.ctx, [fid(j, h) for j, h in groups], [fid(j, k) for j, _ in groups], KR, Kt, aff, cams=cams, counts=True)
            allp = np.concatenate([host[g] for g in groups]); pb = np.cumsum([0] + [len(host[g]) for g in groups]).astype(np.int32)
            st = api.traceOnBatch(W.ctx, [fid(j, k) for j, _ in groups], pb, KR, Kt, aff, allp, cams=cams)
            for i, g in enumerate(groups):
                host[g] = allp[pb[i]:pb[i + 1]].copy(); got, _ = S.get(fid(*g))
                assert got.tobytes() == host[g].tobytes(), (k, g)
                assert np.array_equal(counts[i], _hist(st[pb[i]:pb[i + 1]])) and counts[i].sum() == len(host[g]), (k, g)
                seen |= set(st[pb[i]:pb[i + 1]].tolist())
        if k in (0, 1, 3):
            frames = [fid(j, k) for j in range(n)]
            res, _ = ps.makeNewTracesBatch(list(range(n)), frames, W.clouds(k), W.densities(k), DENS, 1, cap=1 << 15)
            ps.makeNewTracesStore(list(range(n, 2 * n)), frames, W.clouds(k), W.densities(k), DENS, 1, cap=1 << 15)
            for j in range(n):
                host[(j, k)] = _after_make_key_frame(api, *res[j])[0]
                assert S.get(fid(j, k))[0].tobytes() == host[(j, k)].tobytes()
            window.append(k)
    assert {api.IPS_GOOD, api.IPS_OOB, api.IPS_SKIPPED} <= seen, seen
    assert api.traceStoreBatch(W.ctx, [fid(0, 1)], [fid(0, 5)], *[a[None] for a in W.geometry(0, 1, 5)], cams=[MIX[0]]) is None   # no counts: returns without a wait
    W.ctx.sync(); S.drop([fid(j, h) for h in window for j in range(n)])


def test_store_reproduces_reference_trace_new_coarse():
    """the "before" records the reference's running FullSystem held (tests/golden/seq_trace_ref.npz), one block per (frame, host keyframe), all traced in ONE call:
    statuses and every field after the trace equal the reference's"""
    api, synth = _mods(); g = np.load(GOLD); L = int(g["levels"])
    seq = cached_sequence(200, 1000, synth.KITTI_K, synth.KITTI_WH, step=0.5)
    keys = g["keys"]; frames = sorted(set(int(i) for i, _, _ in keys))
    ctx = api.Context(synth.KITTI_K, *synth.KITTI_WH, levels=L, max_frames=len(frames) + 2)
    for i in frames:
        ctx.makeImages(10000 + i, seq.images[i])
    ctx.sync(); S = api.ImmatureStore(ctx)
    o = 0; rec0_all, st0_all, st1_all = g["rec0"], g["st0"].astype(np.int32), g["st1"].astype(np.int32); spans = []
    for j, (i, hidx, m) in enumerate(keys):
        P = np.zeros(m, api.IMMATURE_PT_DTYPE); P.view(np.float32).reshape(m, -1)[:, :29] = rec0_all[o:o + m]; P["lastTraceStatus"] = st0_all[o:o + m]
        S.set(j, P); spans.append((o, m)); o += m
    aff = np.tile(np.array([1.0, 0.0], np.float32), (len(keys), 1))
    counts = api.traceStoreBatch(ctx, np.arange(len(keys)), [10000 + int(i) for i, _, _ in keys], g["KRKi"], g["Kt"], aff, counts=True)
    seen = set()
    for j, (o, m) in enumerate(spans):
        got, _ = S.get(j); st1 = st1_all[o:o + m]
        assert np.array_equal(got["lastTraceStatus"], st1) and np.array_equal(counts[j], _hist(st1)), j
        assert _digest(np.ascontiguousarray(got.view(np.float32).reshape(m, -1)[:, :29]).view(np.uint32)).rstrip(b"\0") == g["rec1_digest"][j], j
        seen |= set(st1.tolist())
    assert len(frames) >= 15 and o > 1500 and {api.IPS_GOOD, api.IPS_OOB, api.IPS_SKIPPED} <= seen
    ctx.close()


def _restate_activation(api, recs, metas, flagged, dec_of, opt_of, cand_rows):
    """FullSystem.cpp:612-720 over host arrays: filter -> (walk decisions, optimize results supplied) -> post pass + swap-with-back compaction"""
    nH = len(recs); cls = []
    for h in range(nH):
        P, M = recs[h], metas[h]; c = np.zeros(len(P), np.int32)
        for i in range(len(P)):
            st = P["lastTraceStatus"][i]
            if M["isFromSensor"][i] == 0 and h == nH - 1: continue
            if not np.isfinite(P["idepth_max"][i]) or st == api.IPS_OUTLIER: c[i] = 1; continue
            can = st in (api.IPS_GOOD, api.IPS_SKIPPED, api.IPS_BADCONDITION, api.IPS_OOB) and P["lastTracePixelInterval"][i] < 8 and P["quality"][i] > np.float32(3) \
                and (P["idepth_max"][i] + P["idepth_min"][i]) > 0
            if not can: c[i] = 1 if (flagged[h] or st == api.IPS_OOB) else 0; continue
            c[i] = 2; cand_rows.append((h, i))
        cls.append(c)
    return cls


def _window(W, j, hosts_k, newest):
    synth = W.synth; c = MIX[j]; K = W.Ks[c]; seq = W.seqs[c]; K0, K1 = orc.distmap_geometry(K, None, None); Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
    def geo(hh):
        R, t = synth.rel_pose(seq.R[hh], seq.t[hh], seq.R[newest], seq.t[newest]); return (K1 @ R.astype(np.float32) @ Ki0).astype(np.float32), (K1 @ t.astype(np.float32)).astype(np.float32)
    G = [geo(h) for h in hosts_k]; cl = seq.clouds[hosts_k[0]][::7]
    uvid = np.stack([np.floor(cl[:, 0]), np.floor(cl[:, 1]), 1.0 / cl[:, 2]], 1).astype(np.float32)
    pre = np.stack([np.concatenate([np.asarray(r, np.float32).reshape(-1), np.asarray(t, np.float32), [1.0, 0.0]]) for h in hosts_k for tt in hosts_k if tt != h
                    for r, t in [synth.rel_pose(seq.R[h], seq.t[h], seq.R[tt], seq.t[tt])]]).astype(np.float32)
    cal = np.array([K[0], K[1], K[2], K[3], 1.0 / K[0], 1.0 / K[1]], np.float32)
    return dict(hosts=[fid(j, h) for h in hosts_k], flagged=[int(j % 2 == 0 and h == hosts_k[0]) for h in hosts_k], cKRKi=np.stack([g[0] for g in G]), cKt=np.stack([g[1] for g in G]),
                pt_begin=[0, len(uvid)], KRKi=G[0][0][None], Kt=G[0][1][None], uvid=uvid, minActDist=1.0 + 0.5 * (j % 3), pre14=pre, calib6=cal)


def test_activation_on_store_equals_host_path(world):
    """activatePointsMT on the store for six mixed sequences (flagged oldest host in half of them, the newest-host rule, non-finite / OUTLIER / OOB / off-image candidates)
    against the host path: sdv_activate_select_batch_cams + sdv_immature_optimize_batch_cams + a numpy restatement of FullSystem.cpp:612-720.  Activated list (order, host,
    index, idepth, res_state), the surviving records and their order per host are identical."""
    W = world; api = W.api; n = len(MIX); S = api.ImmatureStore(W.ctx); ps = api.PixelSelector(W.ctx, n, W.rp, cams=MIX); hk = [0, 1, 3]
    for k in hk:
        ps.makeNewTracesStore(list(range(n)), [fid(j, k) for j in range(n)], W.clouds(k), W.densities(k), DENS, 1, cap=1 << 15)
        if k != 3:
            for kk in (k + 1, k + 2):
                groups = [(j, h) for h in hk if h <= k for j in range(n)]; geo = [W.geometry(j, h, kk) for j, h in groups]
                api.traceStoreBatch(W.ctx, [fid(j, h) for j, h in groups], [fid(j, kk) for j, _ in groups], np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo]),
                                    np.stack([g[2] for g in geo]), cams=[MIX[j] for j, _ in groups])
    seqs = [_window(W, j, hk, 3) for j in range(n)]
    before = {(j, h): S.get(fid(j, h)) for j in range(n) for h in hk}
    got = api.activateStoreBatch(W.ctx, seqs, cams=MIX)
    kinds = set()
    for j in range(n):
        q = seqs[j]; recs = [before[(j, h)][0] for h in hk]; metas = [before[(j, h)][1] for h in hk]; rows = []
        cls = _restate_activation(api, recs, metas, q["flagged"], None, None, rows)
        cb = np.cumsum([0] + [sum(1 for r in rows if r[0] == h) for h in range(3)])
        cand4 = np.array([[recs[h]["u"][i], recs[h]["v"][i], np.float32(0.5) * (recs[h]["idepth_max"][i] + recs[h]["idepth_min"][i]), metas[h]["my_type"][i]] for h, i in rows], np.float32).reshape(-1, 4)
        sq = dict(pt_begin=q["pt_begin"], KRKi=q["KRKi"], Kt=q["Kt"], uvid=q["uvid"], cand_begin=cb, cKRKi=q["cKRKi"], cKt=q["cKt"], cand4=cand4, minActDist=q["minActDist"])
        dec = api.activateSelectBatch(W.ctx, [sq], cams=[MIX[j]])[0]
        opt = [rows[k] for k in range(len(rows)) if dec[k] == 1]
        dead = [np.zeros(len(r), bool) for r in recs]
        for (h, i), d in zip(rows, dec):
            if d == -1: dead[h][i] = True
        for h in range(3):
            dead[h] |= cls[h] == 1
        act = []
        if opt:
            pts = np.concatenate([recs[h][i:i + 1] for h, i in opt]); fs = np.array([metas[h]["isFromSensor"][i] for h, i in opt], np.uint8)
            pb = np.cumsum([0] + [sum(1 for o in opt if o[0] == h) for h in range(3)]); tb = [0, 2, 4, 6]
            st, idp, rs = api.optimizeImmaturePointBatch(W.ctx, pb, tb, [q["hosts"][t] for h in range(3) for t in range(3) if t != h], q["pre14"], np.stack([q["calib6"]] * 3), pts, fs, 1,
                                                         cams=[MIX[j]] * 3)
            for k, (h, i) in enumerate(opt):
                if st[k] == 1: act.append((h, i, idp[k], rs[k, :2]))
                if st[k] in (1, -1) or recs[h]["lastTraceStatus"][i] == api.IPS_OOB: dead[h][i] = True
            kinds |= set(st.tolist())
        assert [a[0] for a in act] == got["host"][j].tolist() and [a[1] for a in act] == got["idx"][j].tolist(), j
        assert np.array_equal(np.array([a[2] for a in act], np.float32), got["idepth"][j]) and np.array_equal(np.array([a[3] for a in act]).reshape(-1, 2), got["res_state"][j]), j
        for k, a in enumerate(act):
            assert got["pts"][j][k].tobytes() == recs[a[0]][a[1]].tobytes() and got["meta"][j][k].tobytes() == metas[a[0]][a[1]].tobytes()
        for h in range(3):
            v = list(range(len(recs[h]))); i = 0
            while i < len(v):
                if dead[h][v[i]]: v[i] = v[-1]; v.pop(); continue
                i += 1
            g, m = S.get(fid(j, hk[h]))
            assert g.tobytes() == recs[h][v].tobytes() and m.tobytes() == metas[h][v].tobytes() and got["counts"][j][h] == len(v), (j, h)
        kinds |= {("del", int((cls[h] == 1).sum() > 0)) for h in range(3)} | {("off", int((dec == -1).any()))}
    assert 1 in kinds and ("del", 1) in kinds and ("off", 1) in kinds, kinds
    S.drop([fid(j, h) for j in range(n) for h in hk])


def test_async_trace_then_release_and_reupload(world):
    """a trace without counts returns before its kernel ran; releasing the traced frame and uploading another image into its storage right away must not change what
    the trace saw: the records equal a trace that waited"""
    W = world; api = W.api; S = api.ImmatureStore(W.ctx); c = MIX[0]
    P = api.immatureInit(W.ctx, fid(0, 0), np.stack([np.arange(20, 1180, 2), np.full(580, 180)], 1), cam=c)
    g = W.geometry(0, 0, 2); args = (g[0][None], g[1][None], g[2][None])
    S.set(9101, P); S.set(9102, P)
    api.traceStoreBatch(W.ctx, [9101], [fid(0, 2)], *args, cams=[c], counts=True)                       # the reference result, waited for
    api.traceStoreBatch(W.ctx, [9102], [fid(0, 2)], *args, cams=[c])                                    # returns at once
    W.ctx._ck(api.LIB.sdv_frame_release(W.ctx.p, fid(0, 2)))
    noise = np.ascontiguousarray(np.random.default_rng(1).uniform(0, 255, (SIZES[c][1], SIZES[c][0])).astype(np.float32))
    W.ctx.makeImagesBatch([fid(0, 2)], [noise.ctypes.data], cams=[c]); W.ctx.sync()
    assert S.get(9102)[0].tobytes() == S.get(9101)[0].tobytes()
    S.drop([9101, 9102])
    img = np.ascontiguousarray(W.seqs[c].images[2], np.float32); W.ctx.makeImagesBatch([fid(0, 2)], [img.ctypes.data], cams=[c]); W.ctx.sync()
