"""Pins the photometric calibration on the reference's own code (oracle/_ref, oracle/gamma.mk), BIT FOR BIT:
  - the host mirror sdv_loam_b200.undistort.PhotometricUndistorter against the reference's PhotometricUndistorter (util/Undistort.cpp:20-214, with a PGM reader in
    place of ImageRW_dummy.cpp): valid, GDepth, getG(), vignetteMapInv and processFrame's output, for settings 0, 1, 2 and every way the constructor fails;
  - orc_gamma.gamma_B against FullSystem::setGammaFunction's CalibHessian::B;
  - the oracle's makeImages with B (orc_gamma.Frame(.., B=B)) against FrameHessian::makeImages(color, &Hcalib) at every level, then makeHists, select / selectFromLidar,
    makeMaps / makeMapsFromLidar and CoarseInitializer::setFirstFromLidar on those frames, with intensities on the x.5 rounding edges of getBGradOnly, beyond both
    clamps, outside the int range, inf and NaN (the conversions the reference leaves undefined; its x86 build gives INT_MIN, so c = 5).
Every case also checks that the weighted result differs from the unweighted one.  The reference's results are stored in tests/golden/ref_pin_gamma.npz
(tests/ref_golden.py); tests/golden/make_gamma_golden.py (SDV_RECORD_REF_GOLDEN=1) re-records them from oracle/_ref."""

import numpy as np
import pytest
import orc
import orc_gamma
import orc_init
import ref
from conftest import cached_sequence, SMALL_K, SMALL_WH
from ref_golden import RefPin

from sdv_loam_b200 import synth
from sdv_loam_b200.undistort import PhotometricUndistorter, write_pgm

EDGE = np.array([4.5, 5.5, 6.5, np.nextafter(np.float32(6.5), np.float32(0)), 100.5, 249.5, 250.5, 251.5, -3.0, 300.0, -2.5e9, 2.5e9, np.inf, -np.inf, np.nan],
                np.float32)


def _ref_gamma():
    import ref_gamma
    return ref_gamma


@pytest.fixture
def pin(request):
    p = RefPin("pin_gamma", request.node.name); yield p; p.save()


def response_text(gamma, n=256, reverse_at=None):
    """the first line of a response file: 255*(i/(n-1))^gamma; reverse_at: a step down there (not strictly increasing)"""
    v = [float(np.float32(255.0 * (i / (n - 1)) ** gamma)) for i in range(n)]
    if reverse_at is not None:
        v[reverse_at] = v[reverse_at - 1]
    return " ".join(repr(x) for x in v) + "\n"


def vignette(wh, bits, seed=0):
    """a radial fall-off, 8- or 16-bit"""
    w, h = wh; y, x = np.mgrid[0:h, 0:w]; r2 = ((x - w / 2) / w) ** 2 + ((y - h / 2) / h) ** 2
    v = np.clip(1.0 - 0.8 * r2 + np.random.default_rng(seed).uniform(-0.01, 0.01, (h, w)), 0.2, 1.0)
    return (v * (255 if bits == 8 else 65535)).astype(np.uint8 if bits == 8 else np.uint16)


PU_CASES = {                                                             # response text, vignette bits (None: missing; "size": wrong size), setting_photometricCalibration
    "g06_v8_pc2": (response_text(0.6), 8, 2), "g16_v16_pc2": (response_text(1.6), 16, 2), "g16_1024_v8_pc1": (response_text(1.6, 1024), 8, 1),
    "g06_v8_pc0": (response_text(0.6), 8, 0), "g16_1024_v16_pc0": (response_text(1.6, 1024), 16, 0),
    "decreasing": (response_text(0.6, reverse_at=100), 8, 2), "short": (response_text(0.6, 200), 8, 2), "no_vignette": (response_text(0.6), None, 2),
    "vignette_size": (response_text(0.6), "size", 2), "no_response": (None, 8, 2),
}


@pytest.mark.parametrize("case", list(PU_CASES))
def test_photometric_undistorter_bit_exact(case, pin, tmp_path):
    text, bits, pc = PU_CASES[case]; wh = (96, 40); w, h = wh
    V = None if bits is None else vignette((w + 3, h) if bits == "size" else wh, 8 if bits == "size" else bits)
    gp, vp = str(tmp_path / "pcalib.txt"), str(tmp_path / "vignette.pgm")
    if text is not None:
        open(gp, "w").write(text)
    if V is not None:
        write_pgm(vp, V)
    mine = PhotometricUndistorter(text, V, w, h, pc)
    assert PhotometricUndistorter.from_files(gp if text is not None else None, vp if V is not None else None, w, h, pc).__dict__.keys() == mine.__dict__.keys()
    R = pin.live(lambda: _ref_gamma().Photometric(gp if text is not None else "", vp if V is not None else "", w, h, pc)); st = pin.live(lambda: R.state())
    assert pin.same(np.int32(mine.valid), lambda: np.int32(st[0]))
    if text is not None:                                                  # without a file the constructor returns before it sets GDepth
        assert pin.same(np.int32(mine.GDepth), lambda: np.int32(st[1]))
    G = mine.getG()
    assert pin.same(np.zeros(0, np.float32) if G is None else G, lambda: np.zeros(0, np.float32) if st[2] is None else st[2])
    if mine.valid:                                                        # an invalid object's vignetteMapInv may be allocated and never written (Undistort.cpp:85-86)
        assert pin.same(mine.vignetteMapInv, lambda: st[3])
    raw = np.random.default_rng(1).integers(0, 256, (h, w)).astype(np.uint8)
    for exposure, factor in ((1.0, 1.0), (0.0, 1.5), (2.0, 0.5)):
        out = mine.processFrame(raw, exposure, factor)
        assert pin.same(out, lambda: R.processFrame(raw, exposure, factor)), (exposure, factor)
    valid = case in ("g06_v8_pc2", "g16_v16_pc2", "g16_1024_v8_pc1", "g06_v8_pc0", "g16_1024_v16_pc0")
    assert mine.valid == valid and (G is None) == (not valid)
    if valid and pc != 0:                                                 # processFrame applies G (and the vignette with setting 2) only then
        assert not np.array_equal(mine.processFrame(raw), raw.astype(np.float32)) and mine.ingest_G is not None
        assert (mine.ingest_vignetteMapInv is not None) == (pc == 2)
    else:
        assert mine.ingest_G is None and mine.ingest_vignetteMapInv is None


def _Gs():
    """the arrays main.cpp hands to setGammaFunction: getG() of valid calibrations (256 and 1024 entries, and both linearised by setting 0), and the identity"""
    out = {}
    for name, (text, bits, pc) in PU_CASES.items():
        G = PhotometricUndistorter(text, vignette((8, 4), 8) if bits is not None else None, 8, 4, pc).getG() if bits in (8, 16) else None
        if G is not None:
            out[name] = G
    out["identity"] = np.arange(256, dtype=np.float32)
    return out


def test_set_gamma_function_bit_exact(pin):
    """orc_gamma.gamma_B = FullSystem::setGammaFunction for every G; the linearised 256-entry G (modes 1 and 2 of main.cpp) and the identity give B[i] = i (gw = 1
    everywhere), the linearised 1024-entry G does not, and NULL leaves B as it was"""
    L = int(pin.value(lambda: ref.set_calib(SMALL_WH[0], SMALL_WH[1], SMALL_K))); ident = np.arange(256, dtype=np.float32)
    Gs = _Gs(); assert len(Gs) == 6
    for name, G in Gs.items():
        B = orc_gamma.gamma_B(G); S = pin.live(lambda: ref.System(L))                        # a fresh FullSystem: CalibHessian B[i] = i
        assert pin.same(B, lambda: _ref_gamma().set_gamma(S, G)), name
        assert np.array_equal(B, ident) == (name in ("g06_v8_pc0", "identity")), name
        if name == "g16_v16_pc2":
            assert pin.same(B, lambda: _ref_gamma().set_gamma(S, None))                 # NULL: setGammaFunction returns at once


def with_edges(img, seed, values=EDGE):
    """`values` at interior lattice pixels 6 px apart; values outside the int range sit in a 3x3 patch of 128 (makeHists' (int) of the square root stays defined)"""
    im = np.array(img, np.float32); h, w = im.shape; rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(8, h - 8, 6), np.arange(8, w - 8, 6), indexing="ij"); pick = rng.permutation(ys.size)[:12 * len(values)]
    for (y, x), v in zip(zip(ys.reshape(-1)[pick], xs.reshape(-1)[pick]), np.tile(values, 12)):
        if not np.isfinite(v) or abs(v) > 1e6:
            im[y - 1:y + 2, x - 1:x + 2] = 128.0
        im[y, x] = v
    return im


CAMS = {"small": (SMALL_WH, SMALL_K, 3000), "kitti": (tuple(synth.KITTI_WH), tuple(synth.KITTI_K), 1000)}


@pytest.mark.parametrize("cam,gamma,n", [("small", 0.6, 256), ("small", 1.6, 1024), ("kitti", 1.6, 256), ("kitti", 0.6, 1024)])
def test_make_images_and_selector_bit_exact(cam, gamma, n, pin):
    wh, K, seed = CAMS[cam]; w, h = wh
    L = int(pin.value(lambda: ref.set_calib(w, h, K)))
    pu = PhotometricUndistorter(response_text(gamma, n), vignette(wh, 8), w, h); G = pu.getG(); B = orc_gamma.gamma_B(G)
    S = pin.live(lambda: ref.System(L)); pin.live(lambda: _ref_gamma().set_gamma(S, G))
    seq = cached_sequence(2, seed, K, wh); rp = orc.libc_random_pattern(w, h); os_ = orc.Selector(w, h, rp); rs = pin.live(lambda: ref.Selector(wh))
    img = with_edges(pu.processFrame(seq.images[0].astype(np.uint8)), seed)
    of, ou = orc_gamma.Frame(img, L, B=B), orc.Frame(img, L)
    rf = pin.live(lambda: ref.Frame(img, wh, L)); pin.live(lambda: _ref_gamma().make_images(S, rf, img))
    for l in range(L):
        assert pin.same(of.absSquaredGrad(l), lambda: rf.absSquaredGrad(l)) and pin.same(of.dI(l), lambda: rf.dI(l)), l
        assert not np.array_equal(of.absSquaredGrad(l), ou.absSquaredGrad(l)) and np.array_equal(of.dI(l), ou.dI(l), equal_nan=True), l
    a, b = os_.makeHists(of); r = pin.live(lambda: rs.makeHists(rf))
    assert pin.same(a, lambda: r[0]) and pin.same(b, lambda: r[1]) and not np.array_equal(a, orc.Selector(w, h, rp).makeHists(ou)[0])
    cloud = seq.clouds[0]; differs = 0
    for pot in (1, 2, 4):
        for th in (1.0, 2.0):
            for c3 in (cloud, None):
                m, n3 = os_.select(of, pot, th, c3); r = pin.live(lambda: rs.select(rf, pot, th, c3))
                assert pin.same(n3, lambda: r[1]) and pin.same(m, lambda: r[0]), (pot, th, c3 is None)
                ou_s = orc.Selector(w, h, rp); ou_s.makeHists(ou); differs += not np.array_equal(m, ou_s.select(ou, pot, th, c3)[0])
    assert differs >= 10, differs
    for start_pot, density in ((3, 500.0), (1, 3000.0), (5, 200.0)):
        for c3 in (cloud, None):
            os_.currentPotential = start_pot; pin.live(lambda: setattr(rs, "currentPotential", start_pot))
            m, k = os_.makeMaps(of, density, 1, 1.0, c3); r = pin.live(lambda: rs.makeMaps(rf, density, 1, 1.0, c3))
            assert pin.same(k, lambda: r[1]) and pin.same(m, lambda: r[0]) and pin.same(os_.currentPotential, lambda: rs.currentPotential), (start_pot, density)
            ou_s = orc.Selector(w, h, rp); ou_s.currentPotential = start_pot
            assert not np.array_equal(m, ou_s.makeMaps(ou, density, 1, 1.0, c3)[0]), (start_pot, density)


@pytest.mark.parametrize("cam,gamma", [("kitti", 0.6), ("kitti", 1.6)])
def test_set_first_from_lidar_bit_exact(cam, gamma, pin):
    """CoarseInitializer::setFirstFromLidar (its makeHists + makeMapsFromLidar run on the weighted absSquaredGrad) on a frame of a calibrated camera"""
    import ref_init
    from test_ref_pin_init import box_of, make_cloud
    wh, K, seed = CAMS[cam]; w, h = wh
    L = int(pin.value(lambda: ref.set_calib(w, h, K)))
    pu = PhotometricUndistorter(response_text(gamma), vignette(wh, 16), w, h); G = pu.getG(); B = orc_gamma.gamma_B(G)
    seq = cached_sequence(2, seed, K, wh); img = with_edges(pu.processFrame(seq.images[0].astype(np.uint8)), seed + 1)
    cloud = make_cloud(seq, "plain"); lrud = box_of(cloud); draws = np.zeros(max(len(cloud), 1), np.int32); rp = orc.libc_random_pattern(w, h)
    o = orc_init.init_from_lidar(orc_gamma.Frame(img, L, B=B), rp, cloud, lrud, 1500.0, draws)
    u = orc_init.init_from_lidar(orc.Frame(img, L), rp, cloud, lrud, 1500.0, draws)
    S = pin.live(lambda: ref.System(L)); pin.live(lambda: _ref_gamma().set_gamma(S, G))
    rf = pin.live(lambda: ref.Frame(img, wh, L)); pin.live(lambda: _ref_gamma().make_images(S, rf, img))
    pnt = pin.live(lambda: ref_init.init_first(S, rf, cloud, lrud))
    assert pin.same(np.int32(o["n_selected"]), lambda: np.int32(len(pnt))) and pin.same(o["pnt"], lambda: pnt)
    assert o["n_selected"] > 50 and not (o["n_selected"] == u["n_selected"] and np.array_equal(o["pnt"], u["pnt"]))
