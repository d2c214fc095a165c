"""tuning probe: the e2e leg of bench.py (RAW mono8 from pinned host memory -> H2D -> Undistort + pyramid -> trackNewestCoarse -> D2H, upload of batch k+1
overlapped with the tracking of batch k): repeated timed passes without a profiler, then one torch.profiler pass that reports per-kernel device time, the busy
time of the H2D copy engine and its idle gaps, and how long the pyramid kernel ran concurrently with track_cluster_kernel (not a test).
usage: python tests/_gpu_prof_e2e.py [B] [batches] [reps] [out.json]; SDV_B200_LIB selects the library"""
import sys, os, json, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import sdv_loam_b200
from sdv_loam_b200 import api
import bench
B = int(sys.argv[1]) if len(sys.argv) > 1 else 1056
NB = int(sys.argv[2]) if len(sys.argv) > 2 else 160
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 3
out = sys.argv[4] if len(sys.argv) > 4 else None
seq, synth = bench.load_sequence()
w, h = seq.wh; ho, wo = seq.raw[1].shape
pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32); rh = np.zeros(len(p4), np.int32)
ctx = api.Context(seq.K, w, h, n_tracker_slots=B, max_frames=3 * B + 16, max_kf_images=12)
ctx.setUndistort(seq.und)
KF = 1 << 40
for b in range(B):
    ctx.makeImages(KF, seq.images[0]); api.CoarseTracker(ctx, b).setCoarseTrackingRef(KF, p4, rh); ctx.releaseFrame(KF)
gts, inits = bench.gt_and_inits(seq, synth, B, bench.N_INIT_POOL, seed=7)
NF = bench.N_FRAMES - 1
host_u8 = torch.empty((NF, B, ho, wo), dtype=torch.uint8, pin_memory=True)
for k in range(NF):
    host_u8[k].copy_(torch.from_numpy(seq.raw[1 + k]).expand(B, ho, wo))
u8_ptrs = [np.uint64(host_u8[k].data_ptr()) + np.arange(B, dtype=np.uint64) * np.uint64(ho * wo) for k in range(NF)]
ids = [np.arange(B, dtype=np.uint64) * 2 + p for p in (0, 1)]
slots = np.arange(B, dtype=np.int32)


def upload(s):
    ctx.makeImagesBatch(ids[s & 1], u8_ptrs[s % NF], raw=True)


def track(s):
    T = inits[(3 * (s // 3) + s % NF) % bench.N_INIT_POOL].copy(); ab = np.zeros((B, 2)); ctx.trackBatch(slots, ids[s & 1], T, ab)   # bench.py init_of: a guess drawn for the frame shown


def leg(first, nb):                                   # bench.py e2e_leg: warm-up 3, then nb timed batches, the last upload charged
    upload(first)
    for s in range(first, first + 3):
        upload(s + 1); track(s)
    ctx.sync(); s1 = first + 3; t0 = time.perf_counter()
    for s in range(s1, s1 + nb):
        if s + 1 < s1 + nb:
            upload(s + 1)
        track(s)
    ctx.sync(); t = time.perf_counter() - t0
    tu = time.perf_counter(); upload(s1 + nb); ctx.sync(); t += time.perf_counter() - tu
    return t, s1 + nb + 1


s = 0; rates = []
for r in range(REPS):
    t, s = leg(s, NB); rates.append(B * NB / t)
lib = os.environ.get('SDV_B200_LIB', 'default')
gbps = [x * ho * wo / 1e9 for x in rates]
print(f"lib={lib} B={B} batches={NB} e2e frames/s " + " ".join(f"{x:.0f}" for x in rates) + "  H2D GB/s " + " ".join(f"{x:.1f}" for x in gbps))

NP = 8
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    leg(s, NP)
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def name(e):
    return e.name.split('(')[0].split('<')[0].replace('void ', '').replace('sdv::', '')


def iv(e):
    return (e.time_range.start, e.time_range.end)


agg = {}
for e in ev:
    a = agg.setdefault(name(e), [0, 0.0]); a[0] += 1; a[1] += (iv(e)[1] - iv(e)[0]) / 1e3
h2d = sorted(iv(e) for e in ev if 'HtoD' in e.name and (iv(e)[1] - iv(e)[0]) > 100)
trk = [iv(e) for e in ev if name(e) == 'track_cluster_kernel']
pyr = [iv(e) for e in ev if name(e).startswith('pyr_')]
span = h2d[-1][1] - h2d[0][0] if h2d else 0.0
busy = sum(b - a for a, b in h2d); gaps = [h2d[i + 1][0] - h2d[i][1] for i in range(len(h2d) - 1)]
ovl = sum(max(0.0, min(p[1], t[1]) - max(p[0], t[0])) for p in pyr for t in trk)
pyr_ms = [(b - a) / 1e3 for a, b in pyr if (b - a) > 50]
print(f"  profiled {NP}+4 batches: H2D copies {len(h2d)} busy {busy/1e3:.2f} ms of span {span/1e3:.2f} ms, idle gaps max {max(gaps)/1e3 if gaps else 0:.3f} ms sum {sum(gaps)/1e3:.2f} ms;"
      f" pyramid kernels overlapping track_cluster_kernel {ovl/1e3:.3f} ms; pyramid kernel ms " + " ".join(f"{x:.3f}" for x in pyr_ms[:12]))
for k, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"  {k:40s} launches {n:5d}  total {ms:9.3f} ms")
if out:
    with open(out, 'w') as f:
        json.dump(dict(lib=lib, B=B, batches=NB, e2e_frames_per_s=rates, h2d_GBps=gbps, h2d_busy_ms=busy / 1e3, h2d_span_ms=span / 1e3, h2d_gap_ms=[g / 1e3 for g in gaps],
                       pyr_track_overlap_ms=ovl / 1e3, pyr_kernel_ms=pyr_ms, kernels={k: dict(launches=n, total_ms=ms) for k, (n, ms) in agg.items()}), f, indent=1)
ctx.close()
