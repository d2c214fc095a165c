"""tuning probe: the e2e leg of bench.py (RAW mono8 from pinned host memory -> H2D -> Undistort + pyramid -> trackNewestCoarse -> D2H) for cameras of
different rectified sizes: every sequence on KITTI-360 (raw 1408x376 -> 1400x360), every sequence on KITTI 00 (1241x376 -> 1200x360), and the sequences
split half/half in ONE context created at 1400x360 with KITTI 00 on camera 1 (sdv_set_camera_size, slots bound with sdv_set_calib_slots_cams, one mixed
raw batch through sdv_frame_upload_batch_raw_u8_cams).  For comparison it also runs two single-size contexts of B/2 sequences each and reports their
combined rate (B frames over the sum of the two times).  The legs alternate in one process; then one torch.profiler pass per leg reports the pyramid kernel's
and track_cluster_kernel's times per batch.  Prints the card name, power limit and SM clock of the same run (not a test).
usage: python tests/_gpu_prof_mixed_sizes.py [B] [batches] [reps] [out.json]; SDV_B200_LIB selects the library"""
import sys, os, json, time, subprocess, types
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
assert B % 2 == 0
K360_CALIB = "Pinhole 552.554261 552.554261 682.049453 238.769549 0\n1408 376\ncrop\n1400 360\n"     # calib/kitti_360.txt of the reference, verbatim
NF = bench.N_FRAMES - 1
seq0, synth = bench.load_sequence()


def drive(name):
    """a raw drive as bench.load_sequence renders KITTI 00's, its rectified K and reference cloud"""
    if name == "kitti":
        seq = seq0
    else:
        u = undistort.Undistort.from_text(K360_CALIB)
        rs = cached_sequence(bench.N_FRAMES, 1360, tuple(float(v) for v in K360_CALIB.split()[1:5]), (u.wOrg, u.hOrg))
        raw = [np.ascontiguousarray(im.astype(np.uint8)) for im in rs.images]
        seq = types.SimpleNamespace(K=u.K4, wh=(u.w, u.h), R=rs.R, t=rs.t, raw=raw, und=u, images=[u.undistort_host(r) for r in raw])
        seq.clouds = [synth.lidar_pixels(synth.World(1360), seq.R[0], seq.t[0], seq.K, seq.wh)]
    pts = synth.select_points(seq.images[0], seq.clouds[0], 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    return seq, p4


drives = {n: drive(n) for n in ("k360", "kitti")}


class Leg:
    """one context at the size of its largest drive; names[b] is the drive of sequence b"""

    def __init__(self, names):
        n = len(names); used = sorted(set(names)); big = "k360" if "k360" in used else "kitti"
        cam = {d: (0 if d == big else 1) for d in used}; self.cam_of = np.array([cam[d] for d in names], np.int32); self.mixed = len(used) > 1
        W, H = drives[big][0].wh
        self.ctx = ctx = api.Context(drives[big][0].K, W, H, n_tracker_slots=n, max_frames=2 * n + 16, max_kf_images=12,
                                       max_ref_points=32768)   # clouds of ~2 000 splats: five resident sets of B sequences fit in 80 GB
        KF = 1 << 40
        for d in used:
            c = cam[d]; sq, p4 = drives[d]
            if c:
                ctx.setCameraSize(c, *sq.wh)
            ctx.setUndistort(sq.und, cam=c)
            sl = np.nonzero(self.cam_of == c)[0].astype(np.int32); ctx.setCalibSlots(sl, [sq.K] * len(sl), cams=[c] * len(sl))
            ctx.makeImages(KF, sq.images[0], cam=c)
            for b in sl:
                api.CoarseTracker(ctx, int(b)).setCoarseTrackingRef(KF, p4, np.zeros(len(p4), np.int32))
            ctx.releaseFrame(KF)
        self.inits = np.zeros((bench.N_INIT_POOL, n, 7))
        for d in used:
            sel = self.cam_of == cam[d]; self.inits[:, sel] = bench.gt_and_inits(drives[d][0], synth, int(sel.sum()), bench.N_INIT_POOL, seed=7)[1]
        raw_of = [drives[d][0].raw for d in names]
        sizes = np.array([r[0].size for r in raw_of], np.uint64)                      # sequences back to back in one pinned buffer per frame
        off = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64); self.bytes = int(sizes.sum())
        self.host = torch.empty((NF, self.bytes), dtype=torch.uint8, pin_memory=True)
        for k in range(NF):
            for b in range(n):
                r = raw_of[b][1 + k].reshape(-1); self.host[k, int(off[b]):int(off[b]) + r.size].copy_(torch.from_numpy(r))
        self.ptrs = [np.uint64(self.host[k].data_ptr()) + off for k in range(NF)]
        self.ids = [np.arange(n, dtype=np.uint64) * 2 + p for p in (0, 1)]
        self.slots = np.arange(n, dtype=np.int32); self.s = 0; self.n = n

    def upload(self, s):
        self.ctx.makeImagesBatch(self.ids[s & 1], self.ptrs[s % NF], raw=True, cams=self.cam_of if self.mixed else None)

    def track(self, s):
        T = self.inits[(3 * (s // 3) + s % NF) % bench.N_INIT_POOL].copy(); ab = np.zeros((self.n, 2)); self.ctx.trackBatch(self.slots, self.ids[s & 1], T, ab)

    def run(self, nb):                                     # bench.py e2e_leg: warm-up 3, then nb timed batches, the last upload charged; returns seconds
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
        return t


def card():
    try:
        dev = torch.cuda.current_device()
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # the card name still comes from torch
        q = f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"
    return q


half = B // 2
legs = {"k360": Leg(["k360"] * B), "kitti": Leg(["kitti"] * B), "split": Leg(["k360"] * half + ["kitti"] * half),
        "k360_half": Leg(["k360"] * half), "kitti_half": Leg(["kitti"] * half)}
secs = {k: [] for k in legs}
for r in range(REPS):
    for k, leg in legs.items():
        secs[k].append(leg.run(NB))
rates = {k: [legs[k].n * NB / t for t in v] for k, v in secs.items()}
rates["two_contexts"] = [B * NB / (a + b) for a, b in zip(secs["k360_half"], secs["kitti_half"])]
gbps = {k: [x * legs[k].bytes / legs[k].n / 1e9 for x in rates[k]] for k in legs}
gbps["two_contexts"] = [(legs["k360_half"].bytes + legs["kitti_half"].bytes) * NB / (a + b) / 1e9 for a, b in zip(secs["k360_half"], secs["kitti_half"])]
lib = os.environ.get('SDV_B200_LIB', 'default'); gpu = card()
print(f"lib={lib} gpu: {gpu}  B={B} batches={NB}")
for k in ("k360", "kitti", "split", "two_contexts"):
    print(f"  {k:12s} e2e frames/s " + " ".join(f"{x:.0f}" for x in rates[k]) + "  H2D GB/s " + " ".join(f"{x:.1f}" for x in gbps[k]))

NP = 8
prof = {}
for k in ("k360", "kitti", "split", "k360_half", "kitti_half"):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
        legs[k].run(NP)
    name = lambda e: e.name.split('(')[0].split('<')[0].replace('void ', '').replace('sdv::', '')
    ev = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    prof[k] = {kn: float(np.median([(e.time_range.end - e.time_range.start) / 1e3 for e in ev if name(e) == kn] or [np.nan])) for kn in ("pyr_fused_kernel", "track_cluster_kernel")}
    print(f"  {k:12s} per batch of {legs[k].n}: pyr_fused_kernel median {prof[k]['pyr_fused_kernel']:.3f} ms, track_cluster_kernel median {prof[k]['track_cluster_kernel']:.3f} ms")
if out:
    with open(out, 'w') as f:
        json.dump(dict(lib=lib, gpu=gpu, B=B, batches=NB, raw_bytes_per_batch={k: l.bytes for k, l in legs.items()}, e2e_frames_per_s=rates, h2d_GBps=gbps,
                       kernel_ms_median=prof), f, indent=1)
for leg in legs.values():
    leg.ctx.close()
