"""Host side of a photometrically calibrated camera, without a GPU or the reference: the PGM reader / writer the vignette goes through, the response line's
parsing (std::istream_iterator<float>: up to the first token that is not a number, each rounded once to float), and what Undistort.set_photometric hands to
Context.setUndistort in each mode (the reference's processFrame applies G with setting_photometricCalibration 1 and 2, the vignette with 2 only)."""
import numpy as np

from sdv_loam_b200.undistort import PhotometricUndistorter, Undistort, _parse_floats, read_pgm, write_pgm
from test_ref_pin_gamma import response_text, vignette


def test_pgm_round_trip(tmp_path):
    for bits in (8, 16):
        v = vignette((37, 11), bits, seed=bits); p = str(tmp_path / f"v{bits}.pgm"); write_pgm(p, v); r = read_pgm(p)
        assert r.dtype == v.dtype and np.array_equal(r, v)


def test_response_line_parsing():
    assert [float(x) for x in _parse_floats("1 2.5 -3e2 x 4")] == [1.0, 2.5, -300.0]
    d = "1.00000005960464477625798673798840354720596224069595336914062"       # 1 + 2^-24 + 2^-60: via double it lands on the midpoint and rounds to 1
    assert _parse_floats(d)[0] == np.nextafter(np.float32(1), np.float32(2)) and np.float32(float(d)) == np.float32(1)
    pu = PhotometricUndistorter(response_text(0.6) + "ignored second line", vignette((4, 3), 8), 4, 3)
    assert pu.valid and pu.GDepth == 256 and pu.getG()[0] == 0 and pu.getG()[255] == 255


def test_set_photometric_per_mode():
    u = Undistort([0.6, 1.8, 0.5, 0.5, 0.0], (64, 32), "none", (64, 32))
    assert u.G is None and u.vignetteMapInv is None
    for pc, has_G, has_V in ((2, True, True), (1, True, False), (0, False, False)):
        pu = PhotometricUndistorter(response_text(1.6), vignette((64, 32), 16), 64, 32, pc); u.set_photometric(pu)
        assert (u.G is not None) == has_G and (u.vignetteMapInv is not None) == has_V and u.photometricUndist is pu and pu.getG() is not None
        if has_G:
            assert u.G.shape == (256,) and np.array_equal(u.G, pu.getG()[:256])
    bad = PhotometricUndistorter(response_text(1.6), None, 64, 32)            # no vignette: invalid, nothing applied, getG() None
    u.set_photometric(bad)
    assert u.G is None and u.vignetteMapInv is None and bad.getG() is None
