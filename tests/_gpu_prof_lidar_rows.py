"""tuning probe: the LiDAR pixel rows on the host against the rows kept in device row sets, for B sequences of the bench's workload (KITTI size, one 64-beam sweep of
the bench's synthetic world per sequence, sweeps back to back in pinned host memory).
  frame step     sdv_lidar_handler_batch (rows copied back, the host carries the box, the call waits) against sdv_lidar_handler_rows_batch + sdv_sync;
                 kernel ms = sdv_last_kernel_ms of the nine front-end kernels (the rows path timed with stats_out, which makes it wait)
  keyframe step  sdv_make_new_traces_store_batch fed the host rows + lidar_density against sdv_make_new_traces_rows_store_batch
Per path: wall ms (host clock around the call; every call ends in a device synchronise), median over the repetitions after one warm-up round; the paths alternate.
Bytes over PCIe per step are computed from shapes.  Prints the card name, power limit and SM clock of the same run (not a test).
usage: python tests/_gpu_prof_lidar_rows.py [B ...] [--reps R] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import ctypes as C
import numpy as np
import torch
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence

CAP_ROWS, CAP_PTS, DENS = 1 << 14, 1 << 11, 600.0


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("B", nargs="*", type=int, default=[132, 1056]); ap.add_argument("--reps", type=int, default=5); ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    w, h = synth.KITTI_WH; K = synth.KITTI_K; seq8 = cached_sequence(8, 2000, K, synth.KITTI_WH)
    sweep = synth.lidar_sweep(synth.World(2000), seq8.R[7], seq8.t[7], seed=4)                 # the bench's keyframe sweep
    img = np.ascontiguousarray(seq8.images[7], np.float32); rp = api.random_pattern(w, h); L = api.LIB
    result = dict(gpu=q, sweep_points=int(len(sweep)), reps=a.reps, runs={})
    for B in a.B:
        ctx = api.Context(K, w, h, max_frames=B + 2); ids = np.arange(1, B + 1, dtype=np.uint64)
        for b0 in range(0, B, 128):
            nb = min(128, B - b0); ctx.makeImagesBatch(ids[b0:b0 + nb], [img.ctypes.data] * nb); ctx.sync()
        fe = api.LidarFrontEnd(ctx); ps = api.PixelSelector(ctx, B, rp); slots = np.arange(B, dtype=np.int32)
        pinned = torch.empty((B * len(sweep), 4), dtype=torch.float32, pin_memory=True).numpy(); pinned[:] = np.tile(sweep, (B, 1))
        sb = (np.arange(B + 1) * len(sweep)).astype(np.int32); lr0 = [[10000, -1, 10000, -1]] * B
        host = fe.handle_packed(pinned, sb, synth.RLC, synth.TLC, K, lr0, cap=CAP_ROWS)
        rows = np.ascontiguousarray(np.concatenate([r["cloud_px"] for r in host])); cb = np.concatenate([[0], np.cumsum([len(r["cloud_px"]) for r in host])]).astype(np.int32)
        dl = np.array([api.lidar_density(r["lrud"], (w, h), DENS) for r in host], np.float32); add = np.array([r["addFeaturePoint"] for r in host], np.int32)
        dd = np.full(B, DENS, np.float32); n_out = np.zeros(B, np.int32); num = np.zeros(2 * B, np.int32)
        def reset():
            for j in range(B): ps.potential(j, 3)
            ctx.sync()
        def t(fn):
            ctx.sync(); t0 = time.perf_counter(); fn(); return 1e3 * (time.perf_counter() - t0)
        runs = {k: [] for k in ("frame_host_rows", "frame_row_sets", "frame_row_sets_stats", "keyframe_host_rows", "keyframe_row_sets")}; kern = {"frame_host_rows": [], "frame_row_sets_stats": []}
        outs = {}
        for rep in range(a.reps + 1):                                                    # round 0 warms up every shape
            ms = t(lambda: fe.handle_packed(pinned, sb, synth.RLC, synth.TLC, K, lr0, cap=CAP_ROWS)); k1 = ctx.last_kernel_ms()
            ms2 = t(lambda: (fe.handleRows(slots, ids, pinned, synth.RLC, synth.TLC, K, cap=CAP_ROWS, sweep_begin=sb), ctx.sync()))
            ms3 = t(lambda: fe.handleRows(slots, ids, pinned, synth.RLC, synth.TLC, K, cap=CAP_ROWS, stats=True, sweep_begin=sb)); k3 = ctx.last_kernel_ms()
            reset(); ms4 = t(lambda: ctx._ck(L.sdv_make_new_traces_store_batch(ctx.p, B, slots, ids, cb, rows.ctypes.data, dl, dd, add, CAP_PTS, n_out, num)))
            outs["host"] = (n_out.copy(), num.copy())
            reset(); ms5 = t(lambda: ctx._ck(L.sdv_make_new_traces_rows_store_batch(ctx.p, B, slots, ids, dd, CAP_PTS, n_out, num)))
            outs["rows"] = (n_out.copy(), num.copy())
            if rep:
                for k, v in zip(runs, (ms, ms2, ms3, ms4, ms5)): runs[k].append(v)
                kern["frame_host_rows"].append(k1); kern["frame_row_sets_stats"].append(k3)
        assert all(np.array_equal(x, y) for x, y in zip(outs["host"], outs["rows"])), "the two keyframe paths disagree"
        med = {k: float(np.median(v)) for k, v in runs.items()}; kmed = {k: float(np.median(v)) for k, v in kern.items()}
        nrows = int(cb[-1]); sweep_b = int(B * sweep.nbytes); row_b = nrows * 24
        r = dict(rows_per_sweep=int(len(host[0]["cloud_px"])), median_wall_ms=med, median_kernel_ms=kmed, points_per_keyframe=int(n_out[0]),
                 pcie_bytes=dict(frame_host_rows=sweep_b + row_b, frame_row_sets=sweep_b, keyframe_host_rows=row_b, keyframe_row_sets=B * 64))
        result["runs"][str(B)] = r
        print(f"B={B:5d} rows/sweep={r['rows_per_sweep']} points/keyframe={r['points_per_keyframe']}")
        for k, v in med.items():
            print(f"   {k:22s} wall {v:9.3f} ms" + (f"   kernel {kmed[k]:8.3f} ms" if k in kmed else "") + (f"   PCIe {r['pcie_bytes'][k] / 1e6:8.1f} MB" if k in r["pcie_bytes"] else ""))
        ctx.close()
    if a.out:
        json.dump(result, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
