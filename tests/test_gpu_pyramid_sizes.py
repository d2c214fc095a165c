"""The one-pass pyramid at sizes whose intermediate levels have an odd width or height: every level bit-exact against the oracle's makeImages through every
ingest source (pinned-host float, device float copied or adopted, device mono8), the packed-texel cache rebuilt after a re-ingest of the same handle, and
trackNewestCoarse against the oracle on such a pyramid.
  1240x372, 4 levels: level 2 is 310x93, level 3 155x46 (the last level-2 row has no child; the last band is short).
  1244x376, 4 levels: w % 4 == 2 (scalar loads), level 1 is 622x188, level 2 311x94, level 3 155x47 (odd level-2 width: its last column has no child)."""
import numpy as np
import pytest
import orc
from conftest import cached_sequence

pytestmark = pytest.mark.gpu
ID7 = np.array([1, 0, 0, 0, 0, 0, 0.0])
SIZES = [(1240, 372), (1244, 376)]
L = 4


def _api():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    return api, synth


def _check_levels(ctx, fid, img):
    f = orc.Frame(img, L); h = img.shape[0]
    for l in range(L):
        dI, ab = ctx.frameLevel(fid, l); oI = f.dI(l); oa = f.absSquaredGrad(l)
        inner = slice(1, (h >> l) - 1)                                      # rows 0 / h-1: dx,dy uninitialised in the reference
        assert np.array_equal(dI[..., 0], oI[..., 0], equal_nan=True), (fid, l)
        assert np.array_equal(dI[inner], oI[inner], equal_nan=True) and np.array_equal(ab[inner], oa[inner], equal_nan=True), (fid, l)


@pytest.mark.parametrize("wh", SIZES)
def test_pyramid_odd_levels_every_source(wh):
    import torch
    api, _ = _api(); w, h = wh
    rng = np.random.default_rng(w + h)
    img = rng.uniform(0, 255, (h, w)).astype(np.float32); img[3, 5] = np.inf; img[h // 2, w // 2] = np.nan
    img8 = rng.integers(0, 256, (h, w)).astype(np.uint8)
    ctx = api.Context((500.0, 500.0, w / 2.0, h / 2.0), w, h, levels=L, max_frames=6)
    ctx.makeImages(1, img); _check_levels(ctx, 1, img)
    d32 = torch.from_numpy(img).cuda(); d8 = torch.from_numpy(img8).cuda(); torch.cuda.synchronize()
    ctx.makeImagesBatch([2], [d32.data_ptr()], device=True); ctx.sync(); _check_levels(ctx, 2, img)
    ctx.makeImagesBatch([3], [d32.data_ptr()], device=True, adopt=True); ctx.sync(); _check_levels(ctx, 3, img)
    ctx.makeImagesBatch([4], [d8.data_ptr()], device=True, u8=True); ctx.sync(); _check_levels(ctx, 4, img8.astype(np.float32))
    ctx.makeImages(1, img8.astype(np.float32)); _check_levels(ctx, 1, img8.astype(np.float32))   # same handle, new image: the packed texels of the old one are gone
    ctx.close()


@pytest.mark.parametrize("wh", SIZES)
def test_track_odd_levels_vs_oracle(wh):
    api, synth = _api(); w, h = wh; K = (718.856, 718.856, w / 2.0 - 12.5, h / 2.0 - 0.5)
    seq = cached_sequence(2, 6000 + w, K, wh)
    pts = synth.select_points(seq.images[0], seq.clouds[0], 2000); p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    rh = np.zeros(len(p4), np.int32)
    ctx = api.Context(K, w, h, levels=L, max_frames=4); ctx.makeImages(0, seq.images[0]); ctx.makeImages(1, seq.images[1])
    tr = api.CoarseTracker(ctx, 0); tr.setCoarseTrackingRef(0, p4, rh, 0.0, 1.0)
    f0, f1 = orc.Frame(seq.images[0], L), orc.Frame(seq.images[1], L)
    otr = orc.CoarseTracker(w, h, L, K); otr.setCoarseTrackingRef(f0, p4, rh, 0.0, 1.0)
    for l in range(L):
        a, b = tr.cloud(l), otr.cloud(l)
        assert len(a[0]) == len(b[0]) > 0 and all(np.array_equal(x, y) for x, y in zip(a, b)), l   # reference colours read from the planar levels
    Tgt = orc.se3_from_rt(*synth.rel_pose(seq.R[0], seq.t[0], seq.R[1], seq.t[1]))
    T0 = orc.se3_mul(orc.se3_exp([0.04, -0.02, 0.05, 0.002, -0.002, 0.001]), Tgt)
    ro = otr.trackNewestCoarse(f1, T0, (0.0, 0.0), L - 1); rg = tr.trackNewestCoarse(1, T0, (0.0, 0.0))
    assert rg["good"] == ro["good"]
    assert np.array_equal(rg["iterations"], ro["iterations"]) and np.array_equal(rg["accepts"], ro["accepts"]) and np.array_equal(rg["evals"], ro["evals"]), (ro, rg)
    assert np.abs(orc.se3_log(orc.se3_mul(rg["T"], orc.se3_inv(ro["T"])))).max() < 1e-5 and np.allclose(rg["ab"], ro["ab"], atol=1e-3)
    assert np.allclose(rg["lastResiduals"], ro["lastResiduals"], rtol=1e-4, equal_nan=True)
    ctx.close()
