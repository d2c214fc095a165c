"""tuning probe: device time of track_cluster_kernel (1 056 jobs) and of the fused refinement (528 jobs) with every slot on the context calibration
against every slot on its own K (three cameras, round-robin over the slots), alternated within one process (not a test)"""
import sys, os, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200
from sdv_loam_b200 import synth, api
import bench
from conftest import cached_sequence

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1056
BR = int(sys.argv[2]) if len(sys.argv) > 2 else 528
REPS = 8
fx, fy, cx, cy = synth.KITTI_K
KS = [tuple(synth.KITTI_K), (721.54, 721.54, 609.56 - 20.5, 172.85 - 8.0), (fx * 1.01, fy * 0.99, cx + 2.0, cy - 2.0)]


def modes(ctx, n):
    slots = np.arange(n, dtype=np.int32)
    own = lambda: ctx.setCalibSlots(slots, [KS[s % 3] for s in slots])
    default = lambda: ctx.clearCalibSlots(slots)
    return [("default", default), ("own", own)]


def track():
    seq, _ = bench.load_sequence(); w, h = seq.wh
    pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32); rh = np.zeros(len(p4), np.int32)
    ctx = api.Context(seq.K, w, h, n_tracker_slots=B, max_frames=B + 2)
    KF = 1 << 40
    for b in range(B):
        ctx.makeImages(KF, seq.images[0]); api.CoarseTracker(ctx, b).setCoarseTrackingRef(KF, p4, rh); ctx.releaseFrame(KF)
    gts, inits = bench.gt_and_inits(seq, synth, B, 6, seed=7)
    for b in range(B):
        ctx.makeImages(b, seq.images[1])
    ctx.sync()
    ms = {"default": [], "own": []}; evals = {}
    for rep in range(2 + REPS):
        for name, apply in modes(ctx, B):
            apply(); T = inits[0].copy(); ab = np.zeros((B, 2))
            r = ctx.trackBatch(list(range(B)), list(range(B)), T, ab)
            if rep >= 2:
                ms[name].append(ctx.last_kernel_ms()); evals[name] = int(r["evals"].sum())
    ctx.close()
    return ms, evals


def refine():
    seq8 = cached_sequence(8, 2000, synth.KITTI_K, synth.KITTI_WH); w, h = synth.KITTI_WH
    pts, hT, hab = synth.make_map(seq8, list(range(7)), n_per_frame=300, seed=2)
    ctx = api.Context(synth.KITTI_K, w, h, n_tracker_slots=BR, max_frames=BR + 9)
    base = 1 << 42; kf_ids = [base + k for k in range(7)]
    for k in range(7):
        ctx.makeImages(kf_ids[k], seq8.images[k])
    rp = api.Reprojector(ctx); slots = np.arange(BR, dtype=np.int32); ids = np.arange(BR, dtype=np.uint64) + np.uint64(base + 100)
    for b in range(BR):
        rp.setMap(b, kf_ids, hT, hab, pts); ctx.makeImages(int(ids[b]), seq8.images[7])
    gt = np.concatenate([synth._quat_from_R(seq8.R[7]), seq8.t[7]]); rng = np.random.default_rng(11)
    order = rng.permutation(rp.n_cells).astype(np.int32)
    T0 = np.stack([synth.se3_mul7(synth.se3_exp7(np.concatenate([rng.normal(0, 0.02, 3), rng.normal(0, 0.001, 3)])), gt) for _ in range(BR)])
    ms = {"default": [], "own": []}; matches = {}
    for rep in range(2 + REPS):
        for name, apply in modes(ctx, BR):
            apply(); r = rp.refineBatch(slots, ids, T0, cell_order=order, max_matches=400)
            if rep >= 2:
                ms[name].append(r["ms"]); matches[name] = float(r["n_matches"].mean())
    ctx.close()
    return ms, matches


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"lib={os.environ.get('SDV_B200_LIB', 'default')} gpu: {gpu}")
for leg, fn, n in (("track_cluster_kernel", track, B), ("refine (reprojectMap + structPoseEstimation)", refine, BR)):
    ms, extra = fn()
    for name in ("default", "own"):
        a = np.array(ms[name])
        print(f"{leg} jobs={n} slots on {name:7s} K: median {np.median(a):.4f} ms  min {a.min():.4f}  max {a.max():.4f}  ({extra[name]})")
