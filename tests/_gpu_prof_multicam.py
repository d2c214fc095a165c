"""tuning probe: the e2e leg of bench.py (RAW mono8 from pinned host memory -> H2D -> Undistort + pyramid -> trackNewestCoarse -> D2H) with every sequence on one
camera (KITTI 00) against the sequences split over the three KITTI cameras (00, 03, 04: raw 1241x376, 1242x375, 1226x370, each camera's own raw drive,
slots bound to its rectified K, one mixed raw batch through sdv_frame_upload_batch_raw_u8_cams).  The two legs alternate in one process; then one
torch.profiler pass per leg reports the pyramid kernel's time per batch.  Prints the card name and power limit of the same run (not a test).
usage: python tests/_gpu_prof_multicam.py [B] [batches] [reps] [out.json]; SDV_B200_LIB selects the library"""
import sys, os, json, time, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, undistort
from conftest import cached_sequence
import bench
B = int(sys.argv[1]) if len(sys.argv) > 1 else 1056
NB = int(sys.argv[2]) if len(sys.argv) > 2 else 160
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 3
out = sys.argv[4] if len(sys.argv) > 4 else None
CALIBS = [bench.KITTI00_CALIB,                                                        # calib/KITTI/00.txt, 03.txt, 04.txt of the reference, verbatim
          "Pinhole 721.5377 721.5377 609.5593 172.854 0\n1242 375\ncrop\n1200 360\n",
          "Pinhole 707.0912 707.0912 601.8873 183.1104 0\n1226 370\ncrop\n1200 360\n"]
NC = len(CALIBS); assert B % NC == 0
NF = bench.N_FRAMES - 1
seq0, synth = bench.load_sequence()


def drive(c):
    """camera c's raw drive as bench.load_sequence renders camera 0's (one seed per camera), its rectified K and reference cloud"""
    u = undistort.Undistort.from_text(CALIBS[c])
    if c == 0:
        seq = seq0
    else:
        import types
        rs = cached_sequence(bench.N_FRAMES, 1000 + c, tuple(float(v) for v in CALIBS[c].split()[1:5]), (u.wOrg, u.hOrg))
        raw = [np.ascontiguousarray(im.astype(np.uint8)) for im in rs.images]
        seq = types.SimpleNamespace(K=u.K4, wh=(u.w, u.h), R=rs.R, t=rs.t, raw=raw, und=u, images=[u.undistort_host(r) for r in raw])
        seq.clouds = [synth.lidar_pixels(synth.World(1000 + c), seq.R[0], seq.t[0], seq.K, seq.wh)]
    pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    return seq, p4


drives = [drive(c) for c in range(NC)]
w, h = seq0.wh


class Leg:
    """one context; cam_of[b] is the camera of sequence b (all 0: the single-camera leg)"""

    def __init__(self, cam_of):
        self.cam_of = np.ascontiguousarray(cam_of, np.int32); self.mixed = bool(self.cam_of.any())
        self.ctx = ctx = api.Context(seq0.K, w, h, n_tracker_slots=B, max_frames=3 * B + 16, max_kf_images=12)
        used = sorted(set(self.cam_of.tolist()))
        for c in used:
            ctx.setUndistort(drives[c][0].und, cam=c)
            sl = np.nonzero(self.cam_of == c)[0].astype(np.int32); ctx.setCalibSlots(sl, [drives[c][0].K] * len(sl))
        KF = 1 << 40
        for c in used:
            ctx.makeImages(KF, drives[c][0].images[0])
            for b in np.nonzero(self.cam_of == c)[0]:
                api.CoarseTracker(ctx, int(b)).setCoarseTrackingRef(KF, drives[c][1], np.zeros(len(drives[c][1]), np.int32))
            ctx.releaseFrame(KF)
        self.inits = np.zeros((bench.N_INIT_POOL, B, 7))
        for c in used:
            sel = self.cam_of == c; self.inits[:, sel] = bench.gt_and_inits(drives[c][0], synth, int(sel.sum()), bench.N_INIT_POOL, seed=7)[1]
        sizes = np.array([drives[c][0].raw[0].size for c in self.cam_of], np.uint64)          # sequences back to back in one pinned buffer per frame
        off = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64); self.bytes = int(sizes.sum())
        self.host = torch.empty((NF, self.bytes), dtype=torch.uint8, pin_memory=True)
        for k in range(NF):
            for b in range(B):
                r = drives[self.cam_of[b]][0].raw[1 + k].reshape(-1); self.host[k, int(off[b]):int(off[b]) + r.size].copy_(torch.from_numpy(r))
        self.ptrs = [np.uint64(self.host[k].data_ptr()) + off for k in range(NF)]
        self.ids = [np.arange(B, dtype=np.uint64) * 2 + p for p in (0, 1)]
        self.slots = np.arange(B, dtype=np.int32); self.s = 0

    def upload(self, s):
        self.ctx.makeImagesBatch(self.ids[s & 1], self.ptrs[s % NF], raw=True, cams=self.cam_of if self.mixed else None)

    def track(self, s):
        T = self.inits[(3 * (s // 3) + s % NF) % bench.N_INIT_POOL].copy(); ab = np.zeros((B, 2)); self.ctx.trackBatch(self.slots, self.ids[s & 1], T, ab)

    def run(self, nb):                                     # bench.py e2e_leg: warm-up 3, then nb timed batches, the last upload charged
        first = self.s; self.upload(first)
        for s in range(first, first + 3):
            self.upload(s + 1); self.track(s)
        self.ctx.sync(); s1 = first + 3; t0 = time.perf_counter()
        for s in range(s1, s1 + nb):
            if s + 1 < s1 + nb:
                self.upload(s + 1)
            self.track(s)
        self.ctx.sync(); t = time.perf_counter() - t0
        tu = time.perf_counter(); self.upload(s1 + nb); self.ctx.sync(); t += time.perf_counter() - tu
        self.s = s1 + nb + 1
        return B * nb / t


def card():
    try:
        dev = torch.cuda.current_device()
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # the card name still comes from torch
        q = f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"
    return q


legs = {"single": Leg(np.zeros(B, np.int32)), "split": Leg(np.repeat(np.arange(NC), B // NC))}
rates = {k: [] for k in legs}
for r in range(REPS):
    for k, leg in legs.items():
        rates[k].append(leg.run(NB))
gbps = {k: [x * legs[k].bytes / B / 1e9 for x in v] for k, v in rates.items()}
lib = os.environ.get('SDV_B200_LIB', 'default'); gpu = card()
print(f"lib={lib} gpu: {gpu}  B={B} batches={NB}")
for k in legs:
    print(f"  {k:6s} raw bytes/batch {legs[k].bytes/1e6:.1f} MB  e2e frames/s " + " ".join(f"{x:.0f}" for x in rates[k]) + "  H2D GB/s " + " ".join(f"{x:.1f}" for x in gbps[k]))

NP = 8
pyr = {}
for k, leg in legs.items():
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        leg.run(NP)
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.name.split('(')[0].split('<')[0].replace('void ', '').replace('sdv::', '').startswith('pyr_')]
    pyr[k] = [(e.time_range.end - e.time_range.start) / 1e3 for e in ev]
    print(f"  {k:6s} pyramid kernel ms per {B}-frame batch: median {np.median(pyr[k]):.3f}  " + " ".join(f"{x:.3f}" for x in pyr[k][:12]))
if out:
    with open(out, 'w') as f:
        json.dump(dict(lib=lib, gpu=gpu, B=B, batches=NB, raw_bytes_per_batch={k: l.bytes for k, l in legs.items()}, e2e_frames_per_s=rates, h2d_GBps=gbps,
                       pyr_kernel_ms=pyr), f, indent=1)
for leg in legs.values():
    leg.ctx.close()
