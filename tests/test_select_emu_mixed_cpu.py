"""Frames of different sizes in one batch of the candidate-management engine (sdv-loam_b200/csrc/sdv_select_core.cuh), run on the CPU through tests/emu/cuda_emu.hpp.
The engine is created at 640x192 (the context size: the random pattern's); the batches interleave 640x192 jobs with 576x160 jobs (w % 32 == 0, h % 32 == 0) and
600x176 jobs (remainders in both: the histogram blocks and the threshold reads past the last block row and column).  Every job must equal the oracle
(oracle/orc_select.cpp, pinned on the reference) run at that job's own size, BIT FOR BIT: makeHists, makeMaps / makeMapsFromLidar, makeNewTraces, distance map and
activation walk."""
import numpy as np
import pytest
import orc
import select_emu as se
import select_emu_mixed as sem
from conftest import cached_sequence, SMALL_K, SMALL_WH

W, H = SMALL_WH
CAMS = [(SMALL_WH, SMALL_K, 3000), ((576, 160), (345.0, 345.0, 280.5, 81.0), 3100), ((600, 176), (360.0, 358.0, 297.0, 88.5), 3200)]
MIX = [0, 1, 2, 1, 0, 2]                                                     # camera of each job of a mixed batch


@pytest.fixture(scope="module")
def scene():
    rp = orc.libc_random_pattern(W, H); cams = []
    for wh, K, seed in CAMS:
        seq = cached_sequence(3, seed, K, wh); L = orc.lib().orc_pyr_levels(*wh); of = [orc.Frame(im, L) for im in seq.images]
        cams.append(dict(wh=wh, K=K, seq=seq, of=of, F=[se.FrameImgs(f) for f in of], rp=orc.libc_random_pattern(*wh)))
    return rp, cams


def test_pattern_of_a_smaller_camera_is_a_prefix():
    """PixelSelector(w_c, h_c) re-seeds with srand(3141592) and draws w_c*h_c bytes: a smaller camera's pattern is the first w_c*h_c bytes of the context's"""
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api
    for (w, h), (wc, hc) in (((640, 192), (576, 160)), ((640, 192), (600, 176)), ((1400, 360), (1200, 360)), ((1400, 360), (1244, 356))):
        big = api.random_pattern(w, h); small = api.random_pattern(wc, hc)
        assert np.array_equal(small, big[:wc * hc]) and np.array_equal(small, orc.libc_random_pattern(wc, hc))


def test_hists_per_size(scene):
    rp, cams = scene; E = sem.MixedEngine(W, H, rp)
    for c in (1, 2, 0):
        C = cams[c]; a, b = E.makeHists(C["F"][0], C["wh"]); oa, ob = orc.Selector(*C["wh"], C["rp"]).makeHists(C["of"][0])
        assert len(a) == (C["wh"][0] // 32) * (C["wh"][1] // 32) and np.array_equal(a, oa) and np.array_equal(b, ob), c


@pytest.mark.parametrize("lidar", [True, False])
def test_make_maps_mixed_batch(scene, lidar):
    """six jobs of three sizes in one batch, different potentials, densities and recursions (up, down, none), with the random sub-selection"""
    rp, cams = scene; E = sem.MixedEngine(W, H, rp)
    pots = [3, 2, 4, 5, 2, 3]; dens = [500., 1500., 60., 2500., 900., 333.]; recs = [1, 1, 1, 1, 0, 1]; ths = [1.0, 1.0, 1.0, 2.0, 1.0, 1.0]
    Fs = [cams[c]["F"][k % 2] for k, c in enumerate(MIX)]; whs = [cams[c]["wh"] for c in MIX]
    clouds = [cams[c]["seq"].clouds[k % 2] for k, c in enumerate(MIX)] if lidar else None
    maps, num, pot, passes = E.makeMaps(Fs, whs, pots, dens, recs, ths, clouds)
    for j, c in enumerate(MIX):
        C = cams[c]; o = orc.Selector(*C["wh"], C["rp"]); o.currentPotential = pots[j]
        m, n = o.makeMaps(C["of"][j % 2], dens[j], recs[j], ths[j], clouds[j] if lidar else None)
        assert n == num[j] and o.currentPotential == pot[j] and np.array_equal(m.astype(np.uint8), maps[j]), (j, c)
    assert set(passes) == {1, 2}


def test_make_new_traces_mixed_batch(scene):
    """two keyframe rounds on slots of three sizes in one batch, addFeaturePoint on for some jobs and off for others: records, ImmaturePoint bytes, numPoints,
    potentials and each slot's persistent map at its own size"""
    rp, cams = scene; E = sem.MixedEngine(W, H, rp); mix = [1, 0, 2]
    slots = [se.Slot(p) for p in (3, 2, 4)]; osel = [orc.Selector(*cams[c]["wh"], cams[c]["rp"]) for c in mix]; omap = [np.zeros(cams[c]["wh"][::-1], np.float32) for c in mix]
    for o, p in zip(osel, (3, 2, 4)): o.currentPotential = p
    dens = [600.0, 1500.0, 300.0]
    for rnd in range(2):
        fr = [rnd, 2 - rnd, rnd + 1]; clouds = [cams[c]["seq"].clouds[fr[j]] for j, c in enumerate(mix)]; whs = [cams[c]["wh"] for c in mix]
        lr = [[int(c[:, 0].min()), int(c[:, 0].max()), int(c[:, 1].min()), int(c[:, 1].max())] for c in clouds]
        dl = [orc.lidar_density(lr[j], whs[j], dens[j]) for j in range(3)]; add = [1, int(rnd == 0), 1]
        outs, imms, num, passes = E.makeNewTraces(slots, [cams[c]["F"][fr[j]] for j, c in enumerate(mix)], whs, clouds, dl, dens, add)
        for j, c in enumerate(mix):
            of = cams[c]["of"][fr[j]]; T, onum, opass = osel[j].makeNewTraces(of, clouds[j], dl[j], dens[j], add[j], omap[j])
            assert T.tobytes() == outs[j].tobytes() and np.array_equal(onum, num[j]) and np.array_equal(opass, passes[j]) and osel[j].currentPotential == slots[j].currentPotential, (rnd, j)
            assert np.array_equal(omap[j].astype(np.uint8), slots[j].map(*whs[j]))
            P = orc.immature_init(of, np.stack([T["u"], T["v"]], 1).astype(np.int32))
            assert P.tobytes() == imms[j].tobytes(), (rnd, j)
            assert len(T) > 50


def test_distance_map_and_activation_walk_mixed(scene):
    """the same sources and candidates walked by sequences of three sizes in one call: each map and each decision equals the oracle's CoarseDistanceMap at that size
    (a candidate inside the large image lies outside a smaller one: decision -1 there)"""
    from test_select_emu_cpu import _distmap_inputs
    rp, cams = scene; E = sem.MixedEngine(W, H, rp); rng = np.random.default_rng(4); seq = cams[0]["seq"]
    pb, KRKi, Kt, uvid = _distmap_inputs(seq, 2, [0, 1], rng)
    cb = [0]; cand = []
    for n in (300, 200):
        u = rng.integers(4, W - 5, n); v = rng.integers(4, H - 5, n); idm = rng.uniform(0.01, 0.4, n).astype(np.float32)
        cand.append(np.stack([u, v, idm, rng.choice([1.0, 2.0, 4.0], n)], 1).astype(np.float32)); cb.append(cb[-1] + n)
    cand = np.concatenate(cand); whs = [cams[c]["wh"] for c in (1, 0, 2)]
    dec, maps = E.activate(whs, pb, KRKi, Kt, uvid, cb, KRKi, Kt, cand, 1.5)
    for j, (w, h) in enumerate(whs):
        od = orc.DistMap(w >> 1, h >> 1); od.make(pb, KRKi, Kt, uvid); do = od.activateSelect(np.array(cb, np.int32), KRKi, Kt, cand, 1.5)
        assert np.array_equal(dec[j], do) and np.array_equal(maps[j], od.get()), (w, h)
        assert (do == 1).sum() > 10
    assert (dec[0] == -1).sum() > (dec[1] == -1).sum()
