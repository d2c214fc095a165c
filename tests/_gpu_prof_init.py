"""measurement: the start of B KITTI sequences on the device (sdv_init_from_lidar_rows_batch: setFirstFromLidar at level 0, the point loop of initializeFromInitializer,
setCTRefForFirstFrame and the one-keyframe map) against the oracle's bootstrap on one host core per sequence.
Every sequence has the bench's keyframe image and one 64-beam sweep of the bench's synthetic world, handled into its row set before the timed calls.
  wall ms    host clock around the call, which ends in a device synchronise; median over the repetitions after one warm-up call
  event ms   sdv_last_kernel_ms: CUDA events from the first to the last work of the call on the tracker stream (host waits between launches included)
  launches   sdv_launch_count difference over one call
  oracle ms  orc_init.init_from_lidar (selection, points, setCoarseTrackingRef) for one sequence on one core, times B
Prints the card name, power limit and SM clocks of the same run (not a test).
usage: python tests/_gpu_prof_init.py [B ...] [--reps R] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
import orc
import orc_init
from conftest import cached_sequence

CAP_PTS, DENS = 1 << 12, 1500.0


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("B", nargs="*", type=int, default=[132, 1056]); ap.add_argument("--reps", type=int, default=5); ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    w, h = synth.KITTI_WH; K = synth.KITTI_K; seq8 = cached_sequence(8, 2000, K, synth.KITTI_WH)
    sweep = synth.lidar_sweep(synth.World(2000), seq8.R[7], seq8.t[7], seed=4)
    img = np.ascontiguousarray(seq8.images[7], np.float32); rp = api.random_pattern(w, h); L = api.LIB
    result = dict(gpu=q, reps=a.reps, runs={})
    for B in a.B:
        ctx = api.Context(K, w, h, n_tracker_slots=B, max_ref_points=1 << 15, max_frames=B + 2); ids = np.arange(1, B + 1, dtype=np.uint64)
        for b0 in range(0, B, 128):
            nb = min(128, B - b0); ctx.makeImagesBatch(ids[b0:b0 + nb], [img.ctypes.data] * nb); ctx.sync()
        fe = api.LidarFrontEnd(ctx); api.PixelSelector(ctx, B, rp); slots = np.arange(B, dtype=np.int32)
        st = fe.handleRows(slots, ids, [sweep] * B, synth.RLC, synth.TLC, K, stats=True); m = st[0]["rows"]
        draws = np.random.default_rng(0).integers(0, 2**31 - 1, size=m, dtype=np.int64).astype(np.int32)
        db = (np.arange(B + 1) * m).astype(np.int32); da = np.ascontiguousarray(np.tile(draws, B)); dd = np.full(B, DENS, np.float32)
        n_out = np.zeros(B, np.int32); n_sel = np.zeros(B, np.int32)
        def call():
            ctx._ck(L.sdv_init_from_lidar_rows_batch(ctx.p, B, slots, ids, dd, db, da, CAP_PTS, n_out, n_sel, None, None, None))
        wall, ev, launches = [], [], []
        for rep in range(a.reps + 1):                                                    # call 0 warms up every shape
            ctx.sync(); l0 = L.sdv_launch_count(ctx.p); t0 = time.perf_counter(); call(); t1 = time.perf_counter()
            if rep:
                wall.append(1e3 * (t1 - t0)); ev.append(ctx.last_kernel_ms()); launches.append(int(L.sdv_launch_count(ctx.p) - l0))
        cl = fe.rows(int(ids[0])); f0 = orc.Frame(img, 4); ot = orc.CoarseTracker(w, h, 4, K); o_ms = []
        for _ in range(3):
            t0 = time.perf_counter(); o = orc_init.init_from_lidar(f0, rp, cl["cloud_px"], cl["lrud"], DENS, draws, tracker=ot); o_ms.append(1e3 * (time.perf_counter() - t0))
        assert np.all(n_out == len(o["pts"])) and np.all(n_sel == o["n_selected"]), "device and oracle disagree"
        r = dict(rows_per_sweep=int(m), n_selected=int(n_sel[0]), points_kept=int(n_out[0]), median_wall_ms=float(np.median(wall)), median_event_ms=float(np.median(ev)),
                 launches_per_call=int(np.median(launches)), wall_ms_per_sequence=float(np.median(wall)) / B, oracle_ms_per_sequence_one_core=float(np.median(o_ms)),
                 oracle_ms_B_sequences_one_core=float(np.median(o_ms)) * B)
        result["runs"][str(B)] = r
        print(f"B={B:5d} rows/sweep={m} numPoints[0]={r['n_selected']} kept={r['points_kept']}  wall {r['median_wall_ms']:9.2f} ms ({r['wall_ms_per_sequence']:.3f} ms/seq)"
              f"  event {r['median_event_ms']:9.2f} ms  launches {r['launches_per_call']}  oracle {r['oracle_ms_per_sequence_one_core']:.2f} ms/seq on one core"
              f" = {r['oracle_ms_B_sequences_one_core']:.0f} ms for B")
        ctx.close()
    if a.out:
        json.dump(result, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
