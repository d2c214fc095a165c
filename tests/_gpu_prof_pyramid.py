"""tuning probe: per-kernel device time of the value leg (adopted resident frames -> pyramid -> trackNewestCoarse) from torch.profiler (not a test).
usage: python tests/_gpu_prof_pyramid.py [B] [batches] [out.json]; SDV_B200_LIB selects the library"""
import sys, os, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import sdv_loam_b200
from sdv_loam_b200 import api
import bench
B = int(sys.argv[1]) if len(sys.argv) > 1 else 1056
NB = int(sys.argv[2]) if len(sys.argv) > 2 else 6
out = sys.argv[3] if len(sys.argv) > 3 else None
seq, synth = bench.load_sequence()
w, h = seq.wh
pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32); rh = np.zeros(len(p4), np.int32)
ctx = api.Context(seq.K, w, h, n_tracker_slots=B, max_frames=2 * B + 2, max_kf_images=12)
KF = 1 << 40
for b in range(B):
    ctx.makeImages(KF, seq.images[0]); api.CoarseTracker(ctx, b).setCoarseTrackingRef(KF, p4, rh); ctx.releaseFrame(KF)
gts, inits = bench.gt_and_inits(seq, synth, B, 6, seed=7)
dev = torch.from_numpy(np.stack([seq.images[1]] * B).astype(np.float32)).cuda()
ptrs = np.uint64(dev.data_ptr()) + np.arange(B, dtype=np.uint64) * np.uint64(h * w * 4)
ids = [np.arange(B, dtype=np.uint64) * 2 + p for p in (0, 1)]
slots = np.arange(B, dtype=np.int32)


def step(s):
    ctx.makeImagesBatch(ids[s & 1], ptrs, device=True, adopt=True)
    T = inits[0].copy(); ab = np.zeros((B, 2)); ctx.trackBatch(slots, ids[s & 1], T, ab)


for s in range(3):
    step(s)
ctx.sync(); torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for s in range(NB):
        step(s)
    ctx.sync(); torch.cuda.synchronize()
agg = {}
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        k = e.name.split('(')[0].split('<')[0].replace('void ', '').replace('sdv::', '')
        a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += e.device_time_total / 1e3
rows = sorted(((k, n, ms, ms / NB) for k, (n, ms) in agg.items()), key=lambda r: -r[2])
lib = os.environ.get('SDV_B200_LIB', 'default')
print(f"lib={lib} B={B} batches={NB}")
for k, n, ms, per in rows:
    print(f"  {k:40s} launches {n:5d}  total {ms:9.3f} ms  per batch {per:8.4f} ms")
if out:
    with open(out, 'w') as f:
        json.dump(dict(lib=lib, B=B, batches=NB, kernels=[dict(name=k, launches=n, total_ms=ms, ms_per_batch=per) for k, n, ms, per in rows]), f, indent=1)
