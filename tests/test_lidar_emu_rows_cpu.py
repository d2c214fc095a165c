"""The LiDAR front-end's device-output path (sdv-loam_b200/csrc/sdv_lidar_core.cuh, LidarEngine::handle_rows: rows written into row-set blocks, the running pixel box
seeded from and written back to per-slot device memory, a header per sweep) run on the CPU through tests/emu/cuda_emu.hpp and compared with the oracle
(orc.LidarFrontEnd, pinned on the reference's own main.cpp by tests/test_ref_pin_lidar.py).  BIT FOR BIT: rows, header, box and addFeaturePoint."""
import numpy as np
import orc
from conftest import SMALL_K, SMALL_WH
from lidar_emu_rows import RowsEngine


def _check_set(E, frame, o):
    """frame's set equals the oracle's handler result o: rows, true count, box, counts, flag, and nothing written past the rows"""
    s = E.sets[frame]; h = s["hdr"]; n = len(o["cloud_px"])
    assert h["rows"] == n and h["overflow"] == 0 and np.array_equal(s["block"][:n], o["cloud_px"]), frame
    assert [h["left"], h["right"], h["up"], h["down"]] == list(o["lrud"]) and (h["numGround"], h["n_segmented"], h["addFeaturePoint"]) == (o["numGround"], o["n_segmented"], o["addFeaturePoint"])
    assert np.isnan(s["block"][n:]).all()


def test_rows_drive_box_on_device():
    """three sequences on slots 2, 0, 1, four consecutive calls (one sweep each per call): the box of each slot lives in "device" memory from call to call; every
    set equals the oracle carrying the box on the host, and the slot's box after the call is the set's snapshot"""
    from test_ref_pin_lidar import sweeps
    synth, S = sweeps(6); fe = orc.LidarFrontEnd(); E = RowsEngine(3); slots = [2, 0, 1]; host_box = {s: [10000, -1, 10000, -1] for s in slots}
    for call in range(4):
        tlc = synth.TLC if call % 2 == 0 else np.array([0.0, -0.08, 0.35]); frames = [100 * s + call for s in slots]; sw = [S[(call + j) % 6] for j in range(3)]
        st = E.handle(slots, frames, sw, synth.RLC, tlc, SMALL_K, SMALL_WH, 1 << 15, stats=(call % 2 == 1))
        for j, s in enumerate(slots):
            o = fe.handle(sw[j], synth.RLC, tlc, SMALL_K, SMALL_WH, host_box[s]); host_box[s] = list(o["lrud"]); n = len(o["cloud_px"])
            _check_set(E, frames[j], o)
            assert n > 3000 and E.boxes[s].tolist() == list(o["lrud"]), (call, s)
            if st is not None:
                assert st[j].tolist() == [n, o["numGround"], o["n_segmented"], o["addFeaturePoint"], 0]


def test_rows_edge_sweeps_and_flag():
    """the empty sweep, NaN-or-near returns, a sparse sweep, and a sweep cut to its lower rings (ground ratio > 0.8: addFeaturePoint 1) — 0/0 gives flag 0 as on the host"""
    from test_ref_pin_lidar import sweeps
    synth, S = sweeps(1, seed0=5); fe = orc.LidarFrontEnd(); E = RowsEngine(4)
    low = S[0][S[0][:, 2] < -1.2]                                                             # returns below the sensor: mostly ground
    cases = [np.zeros((0, 4), np.float32), np.array([[np.nan, 0, 0, 0], [0.01, 0.01, 0, 0]], np.float32), S[0][::7], low]
    st = E.handle([0, 1, 2, 3], [1, 2, 3, 4], cases, synth.RLC, synth.TLC, SMALL_K, SMALL_WH, 1 << 15, stats=True)
    flags = []
    for j, cl in enumerate(cases):
        o = fe.handle(cl, synth.RLC, synth.TLC, SMALL_K, SMALL_WH, [10000, -1, 10000, -1]); _check_set(E, j + 1, o); flags.append(o["addFeaturePoint"])
        assert st[j].tolist() == [len(o["cloud_px"]), o["numGround"], o["n_segmented"], o["addFeaturePoint"], 0]
    assert flags[0] == 0 and flags[3] == 1, flags


def test_rows_128_rings():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import synth
    world = synth.World(3000); R, t = synth.trajectory(1, 3000); sw = synth.lidar_sweep(world, R[0], t[0], beams=128, seed=3)
    args = dict(n_scan=128, horizon=1800, ang_res_x=0.2, ang_res_y=0.427 / 2, ang_bottom=24.9, groundScanInd=100)
    o = orc.LidarFrontEnd(**args).handle(sw, synth.RLC, synth.TLC, SMALL_K, SMALL_WH, [10000, -1, 10000, -1]); E = RowsEngine(1, **args)
    E.handle([0], [7], [sw], synth.RLC, synth.TLC, SMALL_K, SMALL_WH, 1 << 15); _check_set(E, 7, o)
    assert len(o["cloud_px"]) > 6000


def test_rows_overflow_keeps_true_count():
    """cap below the row count: the header keeps the true count and marks the set, the first cap rows are the oracle's, nothing is written past cap; the box and
    the flag are those of the whole sweep"""
    from test_ref_pin_lidar import sweeps
    synth, S = sweeps(1); o = orc.LidarFrontEnd().handle(S[0], synth.RLC, synth.TLC, SMALL_K, SMALL_WH, [10000, -1, 10000, -1]); n = len(o["cloud_px"]); cap = n // 3
    E = RowsEngine(1); st = E.handle([0], [9], [S[0]], synth.RLC, synth.TLC, SMALL_K, SMALL_WH, cap, stats=True); s = E.sets[9]; h = s["hdr"]
    assert h["rows"] == n and h["overflow"] == 1 and st[0].tolist() == [n, o["numGround"], o["n_segmented"], o["addFeaturePoint"], 1]
    assert np.array_equal(s["block"][:cap], o["cloud_px"][:cap]) and np.isnan(s["block"][cap:]).all()
    assert E.boxes[0].tolist() == list(o["lrud"]) and h["addFeaturePoint"] == o["addFeaturePoint"]
