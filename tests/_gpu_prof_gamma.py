"""measurement: the keyframe-rate calls at the bench's shape (B KITTI sequences per call) on four 1200x360 cameras, alternating in one process, every call B jobs of
one camera with the bench's LiDAR rows:
  plain          the bench's keyframe image, no gamma (gw2 table NULL: the kernels without gamma code)
  calibrated     that image through a response 255*(i/255)^0.6 (as processFrame makes it) and sdv_set_gamma_cam with the same response
  unit_table     the calibrated image with the identity response set (the gamma kernels, every weight 1: the same selection as no_gamma)
  no_gamma       the calibrated image without gamma
unit_table against no_gamma is the cost of the table lookup alone; calibrated against no_gamma adds what the weights change in the selection.  The calls:
  hists+maps     sdv_selector_make_maps_batch, makeHists + makeMapsFromLidar (density 600, one recursion), texels cached
  new_traces     sdv_make_new_traces_batch (makeHists, makeMapsFromLidar, makeMaps, Shi-Tomasi typing, ImmaturePoint records), pixel rows from the host
  maps+texels    hists+maps right after a re-ingest of the B frames: includes the packed texels of levels 1..3 (grad_texel_kernel, one gamma lookup per texel)
  init           sdv_init_from_lidar_rows_batch from the frames' row sets
Wall ms: host clock around the call, which ends in a device synchronise; median of the repetitions after one warm-up per camera.
Prints the card name, power limit and SM clocks of the same run (not a test).
usage: python tests/_gpu_prof_gamma.py [--B 132] [--reps 15] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from sdv_loam_b200.undistort import PhotometricUndistorter
from conftest import cached_sequence


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--B", type=int, default=132); ap.add_argument("--reps", type=int, default=15); ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    B = a.B; w, h = synth.KITTI_WH; K = synth.KITTI_K; seq8 = cached_sequence(8, 2000, K, synth.KITTI_WH)
    text = " ".join(repr(float(np.float32(255.0 * (i / 255) ** 0.6))) for i in range(256))
    pu = PhotometricUndistorter(text, np.full((h, w), 200, np.uint8), w, h)
    CAMS = ("plain", "calibrated", "unit_table", "no_gamma"); NC = len(CAMS)
    photo = np.ascontiguousarray(pu.processFrame(seq8.images[7].astype(np.uint8)), np.float32)
    imgs = {0: np.ascontiguousarray(seq8.images[7], np.float32), 1: photo, 2: photo, 3: photo}
    ctx = api.Context(K, w, h, n_tracker_slots=B, max_ref_points=1 << 15, max_frames=NC * B + 2, max_kf_images=8)
    ctx.setGammaFunction(pu.getG(), cam=1); ctx.setGammaFunction(np.arange(256, dtype=np.float32), cam=2)
    ids = {c: np.arange(1 + c * B, 1 + (c + 1) * B, dtype=np.uint64) for c in range(NC)}
    def ingest(c):
        for b0 in range(0, B, 128):
            nb = min(128, B - b0); ctx.makeImagesBatch(ids[c][b0:b0 + nb], [imgs[c].ctypes.data] * nb, cams=[c] * nb)
        ctx.sync()
    for c in range(NC):
        ingest(c)
    rp = api.random_pattern(w, h); ps = api.PixelSelector(ctx, NC * B, rp, cams=[c for c in range(NC) for _ in range(B)]); fe = api.LidarFrontEnd(ctx)
    sweep = synth.lidar_sweep(synth.World(2000), seq8.R[7], seq8.t[7], seed=4)
    slots = {c: np.arange(c * B, (c + 1) * B, dtype=np.int32) for c in range(NC)}
    rows = {}
    for c in range(NC):
        fe.handleRows(slots[c], ids[c], [sweep] * B, synth.RLC, synth.TLC, K, stats=True); rows[c] = fe.rows(int(ids[c][0]))
    cloud = rows[0]["cloud_px"]; m = len(cloud); cloud_all = np.ascontiguousarray(np.tile(cloud, (B, 1))); cbeg = (np.arange(B + 1) * m).astype(np.int32)
    dl = api.lidar_density(rows[0]["lrud"], (w, h), 600.0)
    draws = np.random.default_rng(0).integers(0, 2**31 - 1, size=m, dtype=np.int64).astype(np.int32)
    db = (np.arange(B + 1) * m).astype(np.int32); da = np.ascontiguousarray(np.tile(draws, B)); dd = np.full(B, 1500.0, np.float32)
    n_out = np.zeros(B, np.int32); n_sel = np.zeros(B, np.int32); L = api.LIB
    maps = lambda c: ps.makeMapsBatch(slots[c], ids[c], 600.0, 1, 1.0, clouds=[cloud] * B)
    def init_slots(c):
        ctx.setCalibSlots(list(range(B)), [K] * B, cams=[c] * B)
    calls = {                                                                  # name: (untimed set-up, timed call); init last: its map slots pin the frames
        "hists+maps": (None, maps),
        "new_traces": (None, lambda c: ps.makeNewTracesPacked(list(slots[c]), ids[c], cloud_all, cbeg, dl, 600.0, 1, cap=1 << 11)),
        "maps+texels": (ingest, maps),
        "init": (init_slots, lambda c: ctx._ck(L.sdv_init_from_lidar_rows_batch(ctx.p, B, np.arange(B, dtype=np.int32), ids[c], dd, db, da, 1 << 12, n_out, n_sel, None, None, None))),
    }
    res = dict(gpu=q, B=B, reps=a.reps, ms={})
    for name, (setup, fn) in calls.items():
        t = {c: [] for c in range(NC)}
        for rep in range(a.reps + 1):
            for c in range(NC):
                if setup:
                    setup(c)
                ctx.sync(); t0 = time.perf_counter(); fn(c); ctx.sync(); t1 = time.perf_counter()
                if rep:
                    t[c].append(1e3 * (t1 - t0))
        res["ms"][name] = {CAMS[c]: [float(np.median(t[c])), float(min(t[c])), float(max(t[c]))] for c in range(NC)}     # median, min, max
        print(name, json.dumps(res["ms"][name]))
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
