"""probe (not a test): INTEGRATION.md's three-dataset context (1400x1024, 5 levels; camera 1 KITTI-CARLA 1392x1024, camera 2 KITTI-360 1400x360, camera 3
KITTI 00 1200x360) with and without a frame pool per camera (sdv_set_camera_storage).
- bytes: sdv_camera_storage_bytes per camera with pools, and the cudaMemGetInfo drop around the reservations as a rough cross-check (a shared card's other
  work moves it too);
- time: wall ms per step of raw ingest + trackBatch + refineBatch for S sequences per camera, pools on and off, alternating, REPS repetitions of STEPS steps.
Prints the card name and power limit of the same run.
usage: python tests/_gpu_prof_camera_storage.py [S] [STEPS] [REPS] [out.json]"""
import sys, os, json, time, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth, undistort
from conftest import cached_sequence
from test_undistort import CALIBS

S = int(sys.argv[1]) if len(sys.argv) > 1 else 132
STEPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 3
out = sys.argv[4] if len(sys.argv) > 4 else None
CTX, LEVELS, NF = (1400, 1024), 5, 4
CAMS = {1: "carla", 2: "kitti360", 3: "kitti00"}


def drive(c, name):
    """a raw drive of NF frames (0: keyframe), its Undistort, reference cloud and one-keyframe map"""
    u = undistort.Undistort.from_text(CALIBS[name]); K_raw = tuple(float(v) for v in CALIBS[name].split()[1:5])
    rs = cached_sequence(NF, 4400 + c, K_raw, (u.wOrg, u.hOrg)); raw = [np.ascontiguousarray(im.astype(np.uint8)) for im in rs.images]
    cloud = synth.lidar_pixels(synth.World(4400 + c), rs.R[0], rs.t[0], u.K4, (u.w, u.h)); pts = synth.select_points(u.undistort_host(raw[0]), cloud, 2000)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    mp = np.zeros(len(pts), api.MAP_PT_DTYPE); mp["u"], mp["v"], mp["idepth"] = pts[:, 0], pts[:, 1], pts[:, 2]
    return dict(u=u, raw=raw, p4=p4, map=mp)


drives = {c: drive(c, n) for c, n in CAMS.items()}
I7 = np.array([1.0, 0, 0, 0, 0, 0, 0])


def make(pools):
    n = S * len(CAMS)
    ctx = api.Context(drives[3]["u"].K4, *CTX, levels=LEVELS, n_tracker_slots=n, max_frames=2 if pools else 2 * n + 8, max_kf_images=2, max_ref_points=32768)
    for c, d in drives.items():
        ctx.setCameraSize(c, d["u"].w, d["u"].h); ctx.setUndistort(d["u"], cam=c)
    torch.cuda.synchronize(); free0 = torch.cuda.mem_get_info()[0]
    if pools:
        for c in CAMS:
            ctx.setCameraStorage(c, 2 * S + 2, 2)
    torch.cuda.synchronize(); drop = free0 - torch.cuda.mem_get_info()[0]
    cam_of = np.repeat(list(CAMS), S).astype(np.int32); slots = np.arange(n, dtype=np.int32)
    for c, d in drives.items():
        sl = slots[cam_of == c]; ctx.setCalibSlots(sl, [d["u"].K4] * len(sl), cams=[c] * len(sl))
        kf = 1 << 40 | c; ctx.makeImagesRaw(kf, d["raw"][0], cam=c)
        ctx.setCoarseTrackingRefBatch(sl, [kf] * len(sl), [d["p4"]] * len(sl), [np.zeros(len(d["p4"]), np.int32)] * len(sl))
        rp = api.Reprojector(ctx)
        rp.setMapBatch(sl, [[kf]] * len(sl), [I7[None]] * len(sl), [None] * len(sl), [d["map"]] * len(sl))
    return dict(ctx=ctx, rp=api.Reprojector(ctx), cam_of=cam_of, slots=slots, drop=drop)


def step(L, k):
    ctx, cam_of = L["ctx"], L["cam_of"]; n = len(cam_of)
    ids = np.arange(n, dtype=np.uint64) * 2 + (k & 1)
    ptrs = np.array([drives[c]["raw"][1 + k % (NF - 1)].ctypes.data for c in cam_of], np.uint64)
    ctx.makeImagesBatch(ids, ptrs, raw=True, cams=cam_of)
    T = np.tile(I7, (n, 1)); ab = np.zeros((n, 2))
    ctx.trackBatch(L["slots"], ids, T, ab)
    L["rp"].refineBatch(L["slots"], ids, T, max_matches=150)


def leg_ms(L):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for k in range(STEPS):
        step(L, k)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / STEPS


try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                     # noqa: BLE001
    card = f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"
legs = {p: make(p) for p in (False, True)}
res = dict(card=card, S=S, steps=STEPS, reps=REPS, bytes={}, mem_get_info_drop=legs[True]["drop"])
for c in CAMS:
    fb, kb = legs[True]["ctx"].cameraStorageBytes(c); res["bytes"][c] = dict(frame=fb, kf_image=kb, pool=(2 * S + 2) * fb + 2 * kb)
res["bytes"][0] = dict(zip(("frame", "kf_image"), legs[False]["ctx"].cameraStorageBytes(0)))
res["pool_bytes_total"] = sum(v["pool"] for k, v in res["bytes"].items() if k)
for p in (False, True):
    step(legs[p], 0); step(legs[p], 1)     # warm-up of every shape
t = {False: [], True: []}
for r in range(REPS):
    for p in ((False, True) if r % 2 == 0 else (True, False)):
        t[p].append(leg_ms(legs[p]))
for p, name in ((False, "pools_off"), (True, "pools_on")):
    res[name] = dict(ms_per_step=t[p], median=float(np.median(t[p])), spread=float(max(t[p]) - min(t[p])))
print(json.dumps(res, indent=1))
if out:
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True); json.dump(res, open(out, "w"), indent=1)
for L in legs.values():
    L["ctx"].close()
