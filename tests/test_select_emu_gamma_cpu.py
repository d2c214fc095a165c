"""The candidate-management CUDA source (sdv-loam_b200/csrc/sdv_select_core.cuh) with per-camera gamma weights, run on the CPU through tests/emu/cuda_emu.hpp against
the oracle (orc.Frame with CalibHessian::B, pinned on the reference by tests/test_ref_pin_gamma.py), BIT FOR BIT: gamma_w2 on the rounding edges, beyond the clamps
and for the conversions the reference leaves undefined; makeHists; makeMaps / makeMapsFromLidar and makeNewTraces in batches that mix a calibrated camera, an
uncalibrated one (table NULL) and a camera of another size.  Levels 1 and 2 come in as the packed texels the device's grad_texel_kernel makes (the oracle's
weighted absSquaredGrad); the table weighs level 0 inside the engine.  Intensities outside the int range, inf and NaN appear in the frames of makeHists and makeMaps
only: in makeNewTraces they make Shi-Tomasi scores NaN, whose maximum the reference and the device take differently (a property of makeNewTraces, not of the gamma)."""
import numpy as np
import pytest
import orc
import orc_gamma
import select_emu as se
import select_emu_gamma as sg
from conftest import cached_sequence, SMALL_K, SMALL_WH
from test_ref_pin_gamma import EDGE, response_text, vignette, with_edges

from sdv_loam_b200.undistort import PhotometricUndistorter

W, H = SMALL_WH


def gw2_of(B):
    """the table sdv_set_gamma_cam keeps: gw2[c] = (B[c+1]-B[c])^2, rounded as makeImages rounds gw*gw"""
    B = np.asarray(B, np.float32); gw = B[1:] - B[:-1]; return np.concatenate([gw * gw, [np.float32(1)]]).astype(np.float32)


def c_x86(I):
    """(int)(I+0.5f) as the reference's x86 build computes it (cvttss2si: INT_MIN for NaN and outside the int range), clamped to [5, 250]"""
    t = np.float32(I) + np.float32(0.5)
    c = -2**31 if not (-2.0**31 <= float(t) < 2.0**31) else int(float(t))
    return min(max(c, 5), 250)


@pytest.fixture(scope="module")
def scene():
    cams = []
    for wh, K, seed, gamma, n in ((SMALL_WH, SMALL_K, 3000, 0.6, 256), ((576, 160), (345.0, 345.0, 280.5, 81.0), 3100, None, 0), (SMALL_WH, SMALL_K, 3001, 1.6, 1024)):
        seq = cached_sequence(3, seed, K, wh); L = orc.lib().orc_pyr_levels(*wh)
        if gamma is None:
            B = None; ims = seq.images; big = seq.images[:2]
        else:
            pu = PhotometricUndistorter(response_text(gamma, n), vignette(wh, 16), *wh); B = orc_gamma.gamma_B(pu.getG())
            ims = [with_edges(pu.processFrame(im.astype(np.uint8)), seed + k, EDGE[np.abs(EDGE) < 1e6]) for k, im in enumerate(seq.images)]
            big = [with_edges(pu.processFrame(im.astype(np.uint8)), seed + 7 + k) for k, im in enumerate(seq.images[:2])]
        of = [orc_gamma.Frame(im, L, B=B) for im in ims]; ou = [orc.Frame(im, L) for im in ims]; ofb = [orc_gamma.Frame(im, L, B=B) for im in big]; oub = [orc.Frame(im, L) for im in big]
        cams.append(dict(wh=wh, seq=seq, B=B, gw2=None if B is None else gw2_of(B), of=of, ou=ou, F=[se.FrameImgs(f) for f in of], ofb=ofb, oub=oub,
                         Fb=[se.FrameImgs(f) for f in ofb], rp=orc.libc_random_pattern(*wh)))
    return orc.libc_random_pattern(W, H), cams


def test_gamma_w2_edges():
    B = orc_gamma.gamma_B(PhotometricUndistorter(response_text(1.6), vignette((8, 4), 8), 8, 4).getG()); t = gw2_of(B)
    I = [4.49, 4.5, 5.49, 5.5, np.nextafter(np.float32(6.5), np.float32(0)), 6.5, 100.5, 249.49, 249.5, 250.5, 251.5, 1e3, -3.0, -0.6, -2.5e9, 2.5e9, 3e38, np.inf, -np.inf, np.nan]
    for v in I:
        assert sg.gamma_w2(v, t) == t[c_x86(v)], v
        assert sg.gamma_w2(v, None) == np.float32(1.0), v
    assert {c_x86(v) for v in I} == {5, 6, 7, 101, 249, 250} and c_x86(2.5e9) == 5 and c_x86(np.inf) == 5 and c_x86(np.nan) == 5 and c_x86(1e3) == 250


def test_hists(scene):
    rp, cams = scene; E = sg.GammaEngine(W, H, rp)
    for C in cams:
        for F, of, ou in ((C["F"][0], C["of"][0], C["ou"][0]), (C["Fb"][0], C["ofb"][0], C["oub"][0])):
            a, b = E.makeHists(F, C["wh"], C["gw2"]); oa, ob = orc.Selector(*C["wh"], C["rp"]).makeHists(of)
            assert np.array_equal(a, oa) and np.array_equal(b, ob)
            if C["B"] is not None:
                assert not np.array_equal(a, orc.Selector(*C["wh"], C["rp"]).makeHists(ou)[0])


@pytest.mark.parametrize("lidar", [True, False])
def test_make_maps_mixed(scene, lidar):
    rp, cams = scene; E = sg.GammaEngine(W, H, rp); mix = [0, 1, 2, 0]
    Fs = [cams[c]["Fb"][k % 2] for k, c in enumerate(mix)]; whs = [cams[c]["wh"] for c in mix]; tabs = [cams[c]["gw2"] for c in mix]
    clouds = [cams[c]["seq"].clouds[k % 2] for k, c in enumerate(mix)] if lidar else None
    for dens, rec, th in ((600.0, 1, 1.0), (3000.0, 1, 2.0), (150.0, 0, 1.0)):
        pots = [3, 2, 4, 1]
        maps, num, pot = E.makeMaps(Fs, whs, tabs, pots, [dens] * 4, [rec] * 4, [th] * 4, clouds)
        for j, c in enumerate(mix):
            C = cams[c]; o = orc.Selector(*C["wh"], C["rp"]); o.currentPotential = pots[j]
            m, n = o.makeMaps(C["ofb"][j % 2], dens, rec, th, None if clouds is None else clouds[j])
            assert np.array_equal(maps[j], m.astype(np.uint8)) and num[j] == n and pot[j] == o.currentPotential, (dens, j)
            if C["B"] is not None:
                u = orc.Selector(*C["wh"], C["rp"]); u.currentPotential = pots[j]
                assert not np.array_equal(m, u.makeMaps(C["oub"][j % 2], dens, rec, th, None if clouds is None else clouds[j])[0]), (dens, j)


def test_make_new_traces_mixed(scene):
    rp, cams = scene; E = sg.GammaEngine(W, H, rp); mix = [2, 1, 0]
    slots = [se.Slot() for _ in mix]; osel = [orc.Selector(*cams[c]["wh"], cams[c]["rp"]) for c in mix]; smap = [np.zeros(cams[c]["wh"][::-1], np.float32) for c in mix]
    for k in range(2):
        Fs = [cams[c]["F"][k] for c in mix]; whs = [cams[c]["wh"] for c in mix]; tabs = [cams[c]["gw2"] for c in mix]; cl = [cams[c]["seq"].clouds[k] for c in mix]
        lr = [[int(q[:, 0].min()), int(q[:, 0].max()), int(q[:, 1].min()), int(q[:, 1].max())] for q in cl]
        dl = [orc.lidar_density(lr[j], whs[j], 800.0) for j in range(len(mix))]
        T, num = E.makeNewTraces(slots, Fs, whs, tabs, cl, dl, [800.0] * len(mix), [1] * len(mix), cap=1 << 15)
        for j, c in enumerate(mix):
            To, no, _ = osel[j].makeNewTraces(cams[c]["of"][k], cl[j], dl[j], 800.0, 1, smap[j])
            assert T[j].tobytes() == To.tobytes() and np.array_equal(num[j], no), (k, c)
            if cams[c]["B"] is not None:
                Tu, _, _ = orc.Selector(*cams[c]["wh"], cams[c]["rp"]).makeNewTraces(cams[c]["ou"][k], cl[j], dl[j], 800.0, 1, np.zeros_like(smap[j]))
                assert k or Tu.tobytes() != To.tobytes(), c
