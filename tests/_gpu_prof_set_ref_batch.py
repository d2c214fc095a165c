"""measurement: the keyframe-rate installs for B KITTI sequences — sdv_tracker_set_ref_batch against a loop of sdv_tracker_set_ref, and sdv_map_set_batch against a
loop of sdv_map_set — in the same process, alternating.  Every sequence has the bench's keyframe splats (select_points of the bench's keyframe, HdiF 1e-3,
int(u) rounding) on one shared KITTI keyframe; the mixed batch puts half the slots on a 1400x360 camera of a 1400x360 context.
  wall ms    host clock around the call (each ends in a device synchronise); median over the repetitions after one warm-up call
  launches   sdv_launch_count difference over one call
--parent LIB: n = 1 through sdv_tracker_set_ref of this library and of LIB (another build of the library), alternating in one process.
Prints the card name, power limit and SM clocks of the same run (not a test).
usage: python tests/_gpu_prof_set_ref_batch.py [B ...] [--reps R] [--parent LIB] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
import ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence


def med(f, reps):
    f(); t = []
    for _ in range(reps):
        t0 = time.perf_counter(); f(); t.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(t))


def launches(ctx, f):
    l0 = ctx.launch_count(); f(); return ctx.launch_count() - l0


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("B", nargs="*", type=int, default=[1, 132, 1056]); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent"); ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    w, h = synth.KITTI_WH; K = synth.KITTI_K; seq = cached_sequence(6, 2000, K, synth.KITTI_WH)
    pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32); rh = np.zeros(len(p4), np.int32)
    mp, mT, mab = synth.make_map(seq, [0, 1, 2, 3], n_per_frame=300, seed=2)
    result = dict(gpu=q, reps=a.reps, splats=len(p4), map_points=len(mp), runs={})
    for B in a.B:
        for mixed in ((False, True) if B == 132 else (False,)):
            W = 1400 if mixed else w
            ctx = api.Context(K, W, h, n_tracker_slots=B, max_ref_points=1 << 15, max_frames=8)
            if mixed:                                                       # even slots: camera 1 (1200x360, frame 1); odd slots: camera 0 (1400x360, frame 2)
                ctx.setCameraSize(1, w, h); ctx.setCalibSlots(list(range(0, B, 2)), [K] * len(range(0, B, 2)), cams=[1] * len(range(0, B, 2)))
                ctx.makeImages(1, seq.images[0], cam=1)
                img0 = np.zeros((h, W), np.float32); img0[:, :w] = seq.images[0]; ctx.makeImages(2, img0)
            else:
                ctx.makeImages(1, seq.images[0])
            frames = [1 if (not mixed or b % 2 == 0) else 2 for b in range(B)]
            P4 = []
            for b in range(B):
                P4.append(p4 if frames[b] == 1 else np.ascontiguousarray(p4 + np.array([100, 0, 0, 0], np.float32)))
            R = [rh] * B; slots = list(range(B))
            batch = lambda: ctx.setCoarseTrackingRefBatch(slots, frames, P4, R)
            loop = lambda: [api.CoarseTracker(ctx, b).setCoarseTrackingRef(frames[b], P4[b], rh) for b in range(B)]
            tb, tl = [], []
            for _ in range(2):                                              # alternating
                tb.append(med(batch, a.reps)); tl.append(med(loop, a.reps))
            lb, ll = launches(ctx, batch), launches(ctx, loop)
            key = f"B{B}" + ("_mixed" if mixed else "")
            r = dict(set_ref_batch_ms=min(tb), set_ref_loop_ms=min(tl), launches_batch=lb, launches_loop=ll)
            if not mixed:
                for i in range(4):
                    ctx.makeImages(10 + i, seq.images[i])
                rp = api.Reprojector(ctx); ids = [[10, 11, 12, 13]] * B
                mb = lambda: rp.setMapBatch(slots, ids, [mT] * B, [mab] * B, [mp] * B)
                ml = lambda: [rp.setMap(b, ids[b], mT, mab, mp) for b in range(B)]
                ta, tm = [], []
                for _ in range(2):
                    ta.append(med(mb, a.reps)); tm.append(med(ml, a.reps))
                r.update(map_set_batch_ms=min(ta), map_set_loop_ms=min(tm), map_launches_batch=launches(ctx, mb))
            print(key, json.dumps(r), flush=True); result["runs"][key] = r
            ctx.close()
    if a.parent:                                                            # n = 1 against another build, alternating in one process
        libs = dict(this=api.LIB, parent=C.CDLL(os.path.abspath(a.parent)))
        out = {}
        for name, L in libs.items():
            L.sdv_create.argtypes = [C.POINTER(api.sdv_calib), C.c_int, C.c_int, C.c_int, C.POINTER(api.sdv_settings), C.c_int, C.POINTER(C.c_void_p)]
            L.sdv_frame_upload.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_float]
            L.sdv_tracker_set_ref.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_double, C.c_double]
            L.sdv_tracker_get_cloud.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
            L.sdv_destroy.argtypes = [C.c_void_p]
            s = api.default_settings(); p = C.c_void_p(); cal = api.sdv_calib(*K)
            assert L.sdv_create(C.byref(cal), w, h, 4, C.byref(s), 0, C.byref(p)) == 0
            im = np.ascontiguousarray(seq.images[0], np.float32); assert L.sdv_frame_upload(p, 1, im.ctypes.data, 1.0) == 0
            out[name] = (L, p)
        one = lambda L, p: L.sdv_tracker_set_ref(p, 0, 1, len(p4), p4.ctypes.data, rh.ctypes.data, 0.0, 0.0, 0.0)
        t = {k: [] for k in libs}
        for _ in range(5):
            for k, (L, p) in out.items():
                t[k].append(med(lambda: one(L, p), max(a.reps, 20)))
        clouds = {}
        for k, (L, p) in out.items():
            n = C.c_int(0); L.sdv_tracker_get_cloud(p, 0, 0, C.byref(n), None, None, None, None)
            c4 = [np.zeros(n.value, np.float32) for _ in range(4)]; L.sdv_tracker_get_cloud(p, 0, 0, C.byref(n), *[x.ctypes.data for x in c4]); clouds[k] = np.stack(c4)
        r = dict(n1_this_ms=[round(x, 4) for x in t["this"]], n1_parent_ms=[round(x, 4) for x in t["parent"]],
                 n1_this_median=float(np.median(t["this"])), n1_parent_median=float(np.median(t["parent"])), clouds_equal=bool(clouds["this"].tobytes() == clouds["parent"].tobytes()))
        print("n1", json.dumps(r), flush=True); result["runs"]["n1_vs_parent"] = r
        for k, (L, p) in out.items():
            L.sdv_destroy(p)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
