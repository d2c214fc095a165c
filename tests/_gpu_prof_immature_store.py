"""tuning probe: one per-frame traceNewCoarse step (every candidate of the 7 keyframes of a window traced into the new frame) for B sequences, through the
host-record entry (sdv_immature_trace_batch_cams: records copied to the device and back, stream synchronised) against the immature-point store
(sdv_immature_trace_store_batch: records stay on the device).  KITTI size (1200x360), NPTS candidates per keyframe, left in the state one earlier trace
gives them.  Per path: device ms of the trace kernel (sdv_last_kernel_ms) and wall ms (host clock around the call; the store call is timed with its
per-status counts, which make it wait for the device, and without them followed by sdv_sync), median over the repetitions; the two paths alternate.
Prints the card name, power limit and SM clock of the same run (not a test).
usage: python tests/_gpu_prof_immature_store.py [B ...] [--reps R] [--npts N] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence
from test_ref_pin_trace import candidates
import orc

NH = 7                                                                     # keyframes in the window (setting_maxFrames)


def window(npts):
    """the records of NH host keyframes of one synthetic KITTI drive, each traced once into the next frame, and the geometry of host h -> frame NH"""
    K, wh = tuple(synth.KITTI_K), (1200, 360); seq = cached_sequence(NH + 1, 5500, K, wh)
    ctx = api.Context(K, *wh, max_frames=NH + 2)
    for k in range(NH + 1):
        ctx.makeImages(k, seq.images[k])
    poses = [np.concatenate([synth._quat_from_R(seq.R[k]), seq.t[k]]) for k in range(NH + 1)]; recs, geo = [], []
    for h in range(NH):
        sh = type(seq).__new__(type(seq)); sh.wh = seq.wh; sh.images = [seq.images[h]]
        P = api.immatureInit(ctx, h, candidates(sh, npts, 90 + h)); g1 = orc.trace_geometry(K, poses[h], poses[h + 1])
        api.traceOnBatch(ctx, [h + 1], [0, len(P)], g1[0][None], g1[1][None], g1[2][None], P)
        recs.append(P); geo.append(orc.trace_geometry(K, poses[h], poses[NH]))
    ctx.close()
    return K, wh, seq, recs, geo


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("B", nargs="*", type=int, default=[132, 1056]); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--npts", type=int, default=3300); ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    K, wh, seq, recs, geo = window(a.npts); result = dict(gpu=q, npts=a.npts, hosts=NH, reps=a.reps, runs={})
    for B in a.B:
        ctx = api.Context(K, *wh, max_frames=4); ctx.makeImages(NH, seq.images[NH]); ctx.sync()
        S = api.ImmatureStore(ctx); ng = B * NH
        for b in range(B):
            for h in range(NH):
                S.set(b * NH + h, recs[h])
        host = np.concatenate([recs[h] for _ in range(B) for h in range(NH)]); pb = np.cumsum([0] + [len(recs[h]) for _ in range(B) for h in range(NH)]).astype(np.int32)
        KR = np.stack([geo[h][0] for _ in range(B) for h in range(NH)]); Kt = np.stack([geo[h][1] for _ in range(B) for h in range(NH)])
        aff = np.stack([geo[h][2] for _ in range(B) for h in range(NH)]); frames = [NH] * ng; hosts = np.arange(ng); cams = [0] * ng
        hrec = host.copy(); ctx.sync(); runs = {"host_records": [], "store_counts": [], "store_nowait": []}
        for rep in range(a.reps + 1):                                      # the first round warms up every shape; each round starts from the same records
            hrec[:] = host
            t0 = time.perf_counter(); st = api.traceOnBatch(ctx, frames, pb, KR, Kt, aff, hrec, cams=cams); w = 1e3 * (time.perf_counter() - t0)
            if rep: runs["host_records"].append((ctx.last_kernel_ms(), w))
            for b in range(B):
                for h in range(NH):
                    S.set(b * NH + h, recs[h])
            ctx.sync()
            t0 = time.perf_counter(); cnt = api.traceStoreBatch(ctx, hosts, frames, KR, Kt, aff, cams=cams, counts=True); w = 1e3 * (time.perf_counter() - t0)
            if rep: runs["store_counts"].append((ctx.last_kernel_ms(), w))
            for b in range(B):
                for h in range(NH):
                    S.set(b * NH + h, recs[h])
            ctx.sync()
            t0 = time.perf_counter(); api.traceStoreBatch(ctx, hosts, frames, KR, Kt, aff, cams=cams); ctx.sync(); w = 1e3 * (time.perf_counter() - t0)
            if rep: runs["store_nowait"].append((float("nan"), w))
        hist = np.bincount(st, minlength=6)[:6]
        assert np.array_equal(cnt.sum(0), hist), (cnt.sum(0), hist)                       # the two paths agree on the step they timed
        med = {k: [float(np.median([x[i] for x in v])) for i in range(2)] for k, v in runs.items()}
        r = dict(points=int(pb[-1]), record_bytes_each_way=int(pb[-1]) * api.IMMATURE_PT_DTYPE.itemsize, status_hist=hist.tolist(), median_ms=med)
        result["runs"][str(B)] = r
        print(f"B={B:5d} points={r['points']:9d} ({r['record_bytes_each_way'] / 1e6:.0f} MB of records each way on the host path) statuses={r['status_hist']}")
        for k, (d, w) in med.items():
            print(f"   {k:13s} kernel {d:8.3f} ms   wall {w:8.3f} ms")
        ctx.close()
    if a.out:
        json.dump(result, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
