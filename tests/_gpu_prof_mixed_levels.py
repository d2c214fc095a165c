"""tuning probe: KITTI-CARLA (1392x1024, 5 levels) and KITTI 00 (1200x360, 4 levels) sequences tracked and refined in ONE context created at 1392x1024 x 5
levels with KITTI on camera 1 at its own depth (sdv_set_camera_levels), against two contexts, one per camera.  Per step: one trackNewestCoarse batch over every
sequence (each starts at its camera's depth - 1) and one reprojectMap + structPoseEstimation batch (the refine leg).  The legs alternate in one process;
device-resident frames, host wall time around synchronised calls.  Prints the card name, power limit and SM clock of the same run (not a test).
usage: python tests/_gpu_prof_mixed_levels.py [B] [steps] [reps] [out.json]; SDV_B200_LIB selects the library"""
import sys, os, json, time, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence
import orc
B = int(sys.argv[1]) if len(sys.argv) > 1 else 264
STEPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 3
out = sys.argv[4] if len(sys.argv) > 4 else None
assert B % 2 == 0
CAMS = {"carla": ((957.962, 957.962, 696.0, 512.0), (1392, 1024)), "kitti": (tuple(synth.KITTI_K), tuple(synth.KITTI_WH))}
KFS = [0, 1]


def drive(name, seed):
    K, wh = CAMS[name]; seq = cached_sequence(4, seed, K, wh)
    pts = synth.select_points(seq.images[1], seq.clouds[1], 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    mp, hT, hab = synth.make_map(seq, KFS, n_per_frame=600, seed=1)
    poses = np.array([np.concatenate([synth._quat_from_R(seq.R[i]), seq.t[i]]) for i in range(4)])
    T0 = orc.se3_from_rt(*synth.rel_pose(seq.R[1], seq.t[1], seq.R[2], seq.t[2]))
    return dict(K=K, wh=wh, L=api.pyr_levels(*wh), seq=seq, p4=p4, map=(mp, hT, hab), poses=poses, T0=T0)


drives = {"carla": drive("carla", 8801), "kitti": drive("kitti", 8802)}


class Leg:
    """one context holding the sequences names[b]; camera 0 is the first drive's, camera 1 the second's"""

    def __init__(self, names):
        used = list(dict.fromkeys(names)); n = len(names); d0 = drives[used[0]]
        self.ctx = ctx = api.Context(d0["K"], *d0["wh"], levels=d0["L"], n_tracker_slots=n, max_frames=4 * len(used) + 2, max_kf_images=4, max_ref_points=32768)
        cam = {d: k for k, d in enumerate(used)}; self.n = n
        for d in used:
            c = cam[d]; dv = drives[d]
            if c:
                ctx.setCameraSize(c, *dv["wh"])
            ctx.setCameraLevels(c, dv["L"])
            sl = np.array([b for b in range(n) if names[b] == d], np.int32); ctx.setCalibSlots(sl, [dv["K"]] * len(sl), cams=[c] * len(sl))
            ids = [100 * c + k for k in range(4)]
            ims = [np.ascontiguousarray(im, np.float32) for im in dv["seq"].images]; ctx.makeImagesBatch(ids, [a.ctypes.data for a in ims], cams=[c] * 4); ctx.sync()
            rp = api.Reprojector(ctx)
            for b in sl:
                api.CoarseTracker(ctx, int(b)).setCoarseTrackingRef(ids[1], dv["p4"], np.zeros(len(dv["p4"]), np.int32))
                rp.setMap(int(b), [ids[k] for k in KFS], dv["map"][1], dv["map"][2], dv["map"][0])
        self.rp = rp; self.slots = np.arange(n, dtype=np.int32)
        self.frames = np.array([100 * cam[names[b]] + 2 for b in range(n)], np.uint64)
        self.T0 = np.stack([drives[d]["T0"] for d in names]); self.P = np.stack([drives[d]["poses"][2] for d in names])

    def track(self):
        T = self.T0.copy(); ab = np.zeros((self.n, 2)); self.ctx.trackBatch(self.slots, self.frames, T, ab)

    def refine(self):
        self.rp.refineBatch(self.slots, self.frames, self.P, max_matches=400)

    def run(self, what, steps):
        f = self.track if what == "track" else self.refine
        for _ in range(2):
            f()
        self.ctx.sync(); t0 = time.perf_counter()
        for _ in range(steps):
            f()
        self.ctx.sync(); return (time.perf_counter() - t0) / steps


def card():
    try:
        dev = torch.cuda.current_device()
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"
    return q


half = B // 2
legs = {"one_context": Leg(["carla", "kitti"] * half), "carla_half": Leg(["carla"] * half), "kitti_half": Leg(["kitti"] * half)}
ms = {w: {k: [] for k in legs} for w in ("track", "refine")}
for r in range(REPS):
    for w in ("track", "refine"):
        for k, leg in legs.items():
            ms[w][k].append(1e3 * leg.run(w, STEPS))
for w in ("track", "refine"):
    ms[w]["two_contexts"] = [a + b for a, b in zip(ms[w]["carla_half"], ms[w]["kitti_half"])]
lib = os.environ.get('SDV_B200_LIB', 'default'); gpu = card()
print(f"lib={lib} gpu: {gpu}  B={B} ({half} KITTI-CARLA at 5 levels + {half} KITTI at 4) steps={STEPS}")
for w in ("track", "refine"):
    for k in ("one_context", "two_contexts"):
        print(f"  {w:6s} {k:12s} ms per step " + " ".join(f"{x:.3f}" for x in ms[w][k]))
if out:
    with open(out, 'w') as f:
        json.dump(dict(lib=lib, gpu=gpu, B=B, steps=STEPS, ms_per_step=ms), f, indent=1)
for leg in legs.values():
    leg.ctx.close()
