"""tuning probe: the keyframe-rate stages (LiDAR front-end, makeNewTraces, traceOn of the new candidates into the next frame, distance map + activation walk) for
B sequences in four set-ups: all KITTI-360 (1400x360), all KITTI (1200x360), B/2 of each in ONE 1400x360 context (KITTI on camera 1, every batch interleaved),
and two single-size contexts of B/2 sequences each (their times added).  Per stage: device ms (sdv_last_kernel_ms of the call) and wall ms (host clock around
the call, which ends in a stream synchronise), median over the repetitions.  Prints the card name, power limit and SM clock of the same run (not a test).
usage: python tests/_gpu_prof_keyframe_mixed.py [B] [reps] [out.json]"""
import sys, os, json, time, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence
import orc

B = int(sys.argv[1]) if len(sys.argv) > 1 else 132
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
out = sys.argv[3] if len(sys.argv) > 3 else None
CAM = {"k360": (tuple(synth.K360_K), (1400, 360), 5300), "kitti": (tuple(synth.KITTI_K), (1200, 360), 5400)}


def drive(name):
    K, wh, seed = CAM[name]; seq = cached_sequence(2, seed, K, wh); world = synth.World(seed)
    sweeps = [synth.lidar_sweep(world, seq.R[0], seq.t[0], seed=s) for s in range(4)]
    return dict(K=K, wh=wh, seq=seq, sweeps=sweeps, pat=api.random_pattern(*wh))


D = {n: drive(n) for n in CAM}


class Setup:
    """one context at the size of its largest drive; names[b] is the drive of sequence b"""

    def __init__(self, names):
        used = [n for n in ("k360", "kitti") if n in names]; big = used[0]; self.names = names; n = len(names)
        cam = {d: i for i, d in enumerate(used)}; self.cams = np.array([cam[d] for d in names], np.int32); self.mixed = len(used) > 1
        self.ctx = ctx = api.Context(D[big]["K"], *D[big]["wh"], max_frames=8, max_kf_images=8)
        for d in used:
            c = cam[d]
            if c:
                ctx.setCameraSize(c, *D[d]["wh"])
            for k in range(2):
                ctx.makeImages(10 * c + k, D[d]["seq"].images[k], cam=c)
        self.ps = api.PixelSelector(ctx, n, D[big]["pat"], cams=self.cams if self.mixed else None); self.fe = api.LidarFrontEnd(ctx)
        sw = [D[d]["sweeps"][b % 4] for b, d in enumerate(names)]; self.sb = np.concatenate([[0], np.cumsum([len(s) for s in sw])]).astype(np.int32)
        self.xyzi = np.ascontiguousarray(np.concatenate(sw), np.float32); self.K4 = np.array([D[d]["K"] for d in names], np.float32)
        self.cm = self.cams if self.mixed else None

    def stages(self):
        """one keyframe step of every sequence -> {stage: (device ms, wall ms)}"""
        ctx, n, r = self.ctx, len(self.names), {}
        def timed(name, f):
            t0 = time.perf_counter(); v = f(); r[name] = (ctx.last_kernel_ms(), 1e3 * (time.perf_counter() - t0)); return v
        lid = timed("lidar", lambda: self.fe.handle_packed(self.xyzi, self.sb, synth.RLC, synth.TLC, self.K4, [[10000, -1, 10000, -1]] * n, cams=self.cm))
        cl = [x["cloud_px"] for x in lid]; cb = np.concatenate([[0], np.cumsum([len(c) for c in cl])]).astype(np.int32); allc = np.ascontiguousarray(np.concatenate(cl))
        dl = [api.lidar_density(x["lrud"], D[d]["wh"], 1500.0) for x, d in zip(lid, self.names)]
        res, _ = timed("new_traces", lambda: self.ps.makeNewTracesPacked(list(range(n)), [10 * int(c) for c in self.cams], allc, cb, dl, 1500.0, 1, cap=1 << 14))
        pts = np.concatenate([x[1] for x in res]).copy(); pb = np.cumsum([0] + [len(x[1]) for x in res]).astype(np.int32)
        geo = {d: orc.trace_geometry(D[d]["K"], np.concatenate([synth._quat_from_R(D[d]["seq"].R[0]), D[d]["seq"].t[0]]),
                                     np.concatenate([synth._quat_from_R(D[d]["seq"].R[1]), D[d]["seq"].t[1]])) for d in set(self.names)}
        g = [geo[d] for d in self.names]
        timed("trace", lambda: api.traceOnBatch(ctx, [10 * int(c) + 1 for c in self.cams], pb, np.stack([x[0] for x in g]), np.stack([x[1] for x in g]), np.stack([x[2] for x in g]), pts, cams=self.cm))
        seqs = []
        for b, d in enumerate(self.names):
            K0, K1 = orc.distmap_geometry(D[d]["K"], None, None); A = (K1 @ np.linalg.inv(K0.astype(np.float64)).astype(np.float32)).astype(np.float32); z = np.zeros(3, np.float32)
            c = cl[b][::4]; p = pts[pb[b]:pb[b + 1]]; good = p["lastTraceStatus"] == api.IPS_GOOD
            cand = np.stack([p["u"][good], p["v"][good], 0.5 * (p["idepth_max"][good] + p["idepth_min"][good]), np.ones(good.sum())], 1).astype(np.float32)
            seqs.append(dict(pt_begin=[0, len(c)], KRKi=A[None], Kt=z[None], uvid=np.stack([np.floor(c[:, 0]), np.floor(c[:, 1]), 1.0 / c[:, 2]], 1).astype(np.float32),
                             cand_begin=[0, len(cand)], cKRKi=A[None], cKt=z[None], cand4=cand, minActDist=2.0))
        P = api.packActivation(seqs, self.cm)
        timed("activation", lambda: api.activateSelectPacked(ctx, P))
        return r


def med(runs):
    return {k: tuple(float(np.median([x[k][i] for x in runs])) for i in range(2)) for k in runs[0]}


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    h = B // 2
    setups = {"all_k360": [Setup(["k360"] * B)], "all_kitti": [Setup(["kitti"] * B)], "mixed_one_ctx": [Setup(["k360", "kitti"] * h)],
              "two_ctx": [Setup(["k360"] * h), Setup(["kitti"] * h)]}
    runs = {k: [] for k in setups}
    for rep in range(REPS + 1):                                            # the set-ups alternate; the first round warms up every shape
        for k, ss in setups.items():
            rs = [s.stages() for s in ss]
            if rep:
                runs[k].append({st: tuple(sum(r[st][i] for r in rs) for i in range(2)) for st in rs[0]})
    result = dict(gpu=q, B=B, reps=REPS, stages={k: med(v) for k, v in runs.items()})
    for k, v in result["stages"].items():
        print(f"{k:14s} " + "  ".join(f"{st} {d:7.3f}/{w:7.3f} ms" for st, (d, w) in v.items()) + f"   total {sum(x[0] for x in v.values()):.3f}/{sum(x[1] for x in v.values()):.3f} ms")
    if out:
        json.dump(result, open(out, "w"), indent=1)


if __name__ == "__main__":
    main()
