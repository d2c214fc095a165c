"""Pins the restatement of the start of a sequence (oracle/orc_init.cpp: CoarseInitializer::setFirstFromLidar at level 0, the point loop of
FullSystem::initializeFromInitializer and CoarseTracker::setCTRefForFirstFrame) on the reference's own compiled CoarseInitializer.cpp / FullSystem.cpp /
CoarseTracker.cpp (oracle/_ref), one member at a time: BIT FOR BIT.  The reference's results are stored in tests/golden/ref_pin_init.npz (tests/ref_golden.py);
SDV_RECORD_REF_GOLDEN=1 re-records them from oracle/_ref.
Compared: numPoints[0], the Pnt list (u, v, my_type, mdepth, isFromSensor), which points are kept, every PointHessian field the device records carry, and the
tracker's clouds (pc_u, pc_v, pc_idepth, pc_color, pc_n) at every level.  Not compared: PointHessian::type, which the reference leaves uninitialised here.
Rows stay 20 px from the border (tests/seq_replay.py): setFirstFromLidar's dead levels >= 1 read the pattern around every row without a bounds check."""
import ctypes as C

import numpy as np
import pytest
import orc
import orc_init
import ref
import ref_init
from conftest import cached_sequence
from ref_golden import RefPin
from seq_replay import frame_cloud

from sdv_loam_b200 import synth

CASES = {                                                                     # wh, K, sequence seed
    "kitti": (tuple(synth.KITTI_WH), tuple(synth.KITTI_K), 1000),
    "kitti360": ((1400, 360), tuple(synth.K360_K), 1100),
    "carla": ((1392, 1024), (957.962, 957.962, 696.0, 512.0), 1200),        # KITTI-CARLA, 5 levels
}


def rand_after(seed, n):
    """rand() of the C library after srand(seed): what initializeFromInitializer draws after ref_sys_init_from_initializer's srand"""
    libc = C.CDLL(None); libc.srand(seed)
    return np.array([libc.rand() for _ in range(n)], np.int32)


def box_of(cloud):
    """FullSystem::left, right, up, down as lidarCloudHandler grows them from the box of the sweep's pixels (main.cpp:840-847)"""
    if len(cloud) == 0:
        return np.array([10000, -1, 10000, -1], np.int32)
    return np.array([int(cloud[:, 0].min()), int(cloud[:, 0].max()), int(cloud[:, 1].min()), int(cloud[:, 1].max())], np.int32)


def make_cloud(seq, variant):
    """frame 0's pixel rows (20 px from the border), and the case's changes"""
    cl = frame_cloud(seq, 0).copy()
    if variant == "nonpositive":                                              # rows with depth <= 0 among the selected ones
        cl[::7, 2] = 0.0; cl[3::11, 2] = -1.5
    if variant == "collide":                                                  # two rows that round to the same splat pixel: the ordered sums of makeCoarseDepthForFirstFrame
        extra = cl[::5].copy(); extra[:, :2] += 0.2; extra[:, 2] *= 1.37
        cl = np.concatenate([cl, extra])
    if variant == "empty":
        cl = cl[:0]
    return np.ascontiguousarray(cl, np.float64)


@pytest.fixture
def pin(request):
    p = RefPin("pin_init", request.node.name); yield p; p.save()


@pytest.mark.parametrize("cam,variant,density,small_box", [
    ("kitti", "plain", 300.0, False), ("kitti", "plain", 1e6, False), ("kitti", "nonpositive", 500.0, False), ("kitti", "collide", 2000.0, False),
    ("kitti", "plain", 40.0, True), ("kitti", "empty", 2000.0, False),
    ("kitti360", "plain", 700.0, False), ("kitti360", "collide", 1e6, True),
    ("carla", "plain", 1500.0, False), ("carla", "nonpositive", 1e6, False)])
def test_init_from_lidar_bit_exact(cam, variant, density, small_box, pin):
    wh, K, seed = CASES[cam]; w, h = wh
    L = int(pin.value(lambda: ref.set_calib(w, h, K)))
    seq = cached_sequence(2, seed, K, wh)
    cloud = make_cloud(seq, variant)
    lrud = box_of(cloud)
    if small_box:                                                             # a box far smaller than the sweep: density 0.03*area is low and makeMapsFromLidar recurses
        lrud = np.array([lrud[0], lrud[0] + 160, lrud[2], lrud[2] + 40], np.int32)
    draw_seed = 4242 + seed
    draws = rand_after(draw_seed, max(len(cloud), 1))
    rp = orc.libc_random_pattern(w, h)
    f0 = orc.Frame(seq.images[0], L); ot = orc.CoarseTracker(w, h, L, K)
    o = orc_init.init_from_lidar(f0, rp, cloud, lrud, density, draws, tracker=ot)

    S = pin.live(lambda: ref.System(L)); r0 = pin.live(lambda: ref.Frame(seq.images[0], wh, L)); r1 = pin.live(lambda: ref.Frame(seq.images[1], wh, L))
    pnt = pin.live(lambda: ref_init.init_first(S, r0, cloud, lrud))
    ns = o["n_selected"]
    assert pin.same(np.int32(ns), lambda: np.int32(len(pnt)))
    assert pin.same(o["pnt"], lambda: pnt)
    ph = pin.live(lambda: ref_init.init_from_initializer(S, r1, draw_seed, density))
    kept = o["pts"]; k = len(kept)
    # keep decisions: the kept Pnts, in order, at the pixel their ImmaturePoint got
    kuv = np.stack([(o["pnt"][o["keep"] == 1, 0] + np.float32(0.5)).astype(np.int32), (o["pnt"][o["keep"] == 1, 1] + np.float32(0.5)).astype(np.int32)], 1).astype(np.float32)
    assert pin.same(kuv.reshape(-1, 2), lambda: ph[:, :2])
    if variant != "empty":
        assert 0 < k and (density > 1e5 or k < ns), (k, ns)                    # a real keep test below numPoints[0], everything above
    # the PointHessian fields the records carry: u, v, idepth, idepth_zero, idepth_scaled, my_type, energyTH, hasDepthPrior, isFromSensor, status (ACTIVE), color, weights
    mine = np.zeros((k, 26), np.float32)
    mine[:, 0], mine[:, 1] = kept["u"], kept["v"]; mine[:, 2] = mine[:, 3] = mine[:, 4] = o["idepth"]
    mine[:, 5] = o["meta"]["my_type"]; mine[:, 6] = kept["energyTH"]; mine[:, 7] = 1; mine[:, 8] = o["meta"]["isFromSensor"]; mine[:, 9] = 0
    mine[:, 10:18] = kept["color"]; mine[:, 18:26] = kept["weights"]
    assert pin.same(mine, lambda: ph)
    assert np.array_equal(kept["idepth_min"], o["idepth"]) and np.array_equal(kept["idepth_max"], o["idepth"]) and np.all(o["meta"]["type"] == 0)
    rt = pin.live(lambda: ref.CoarseTracker()); pin.live(lambda: ref_init.tracker_set_first(S, rt))
    for lvl in range(L):
        mc = ot.cloud(lvl)
        assert pin.same(np.int32(len(mc[0])), lambda: np.int32(len(rt.cloud(lvl)[0]))), lvl
        assert pin.same(np.stack(mc, 1), lambda: np.stack(rt.cloud(lvl), 1)), lvl
        if variant == "empty":
            assert len(mc[0]) == 0


def reference_start():
    """tests/golden/seq_init_ref.npz: the reference's own FullSystem over frames 0 and 1 of S-KITTI-200 (srand(seed) before frame 1), and the inputs to replay it:
    frames 0 and 1, the rand() draws of initializeFromInitializer (the C library's stream after srand(seed)) and the Reprojector's cell order, which continues that
    stream numPoints[0] draws later"""
    import os
    from sdv_loam_b200 import synth
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seq_init_ref.npz")))
    seq = cached_sequence(2, 1000, synth.KITTI_K, synth.KITTI_WH, step=0.5)               # the first two frames of S-KITTI-200
    assert np.array_equal(frame_cloud(seq, 0), g["rows0"])
    seed = int(g["seed"]); draws = rand_after(seed, len(g["rows0"]))
    libc = C.CDLL(None); libc.srand(seed)
    for _ in range(int(g["n_selected"])):
        libc.rand()
    n_cells = int(np.ceil(seq.wh[0] / 25.0)) * int(np.ceil(seq.wh[1] / 25.0))
    order = np.array(ref.libc_rand_shuffle(n_cells), np.int32)                            # std::random_shuffle on the continuing stream (Reprojector.cpp:107)
    return g, seq, draws, order


def test_oracle_follows_the_reference_run():
    """the oracle's bootstrap on frame 0's rows gives the reference run's numPoints[0], and its trackNewCoarse of frame 1 the reference's pose (1e-3 m / rad) and
    energy (1e-4 relative): the draws and the cell order are where a running reference takes them from"""
    from sdv_loam_b200 import synth
    g, seq, draws, order = reference_start(); w, h = seq.wh; K = tuple(synth.KITTI_K); L = int(g["levels"]); T0 = np.array([1, 0, 0, 0, 0, 0, 0.0])
    f0, f1 = orc.Frame(seq.images[0], L), orc.Frame(seq.images[1], L); ot = orc.CoarseTracker(w, h, L, K); ot.settings(6.0, 20.0, -1.0, -1.0)
    o = orc_init.init_from_lidar(f0, orc.libc_random_pattern(w, h), g["rows0"], g["lrud0"], 1500.0, draws, tracker=ot)
    assert o["n_selected"] == int(g["n_selected"])
    mp = np.zeros(len(o["pts"]), [("u", "<f4"), ("v", "<f4"), ("idepth", "<f4"), ("host", "<i4"), ("type", "<i4")])
    mp["u"], mp["v"], mp["idepth"] = o["pts"]["u"], o["pts"]["v"], o["idepth"]
    r = orc.track_new_coarse(ot, f1, K, [f0], T0.reshape(1, 7), np.zeros((1, 2)), mp, T0, T0, T0, [0.0, 0.0], 2, np.full(5, 100.0), cell_order=order)
    d = orc.se3_log(orc.se3_mul(r["camToTrackingRef"], orc.se3_inv(g["camToTrackingRef"])))
    assert np.abs(d).max() < 1e-3, d
    assert abs(r["lastCoarseRMSE"][0] - g["lastCoarseRMSE"][0]) <= 1e-4 * g["lastCoarseRMSE"][0], (r["lastCoarseRMSE"], g["lastCoarseRMSE"])
    assert np.allclose(r["aff_g2l"], g["aff_g2l"], atol=1e-9)
