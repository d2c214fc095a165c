"""measurement: the back-end keyframe step around optimize_batch for B windows of the bench's shape (7 KITTI keyframes, about 1 700 points and 8 300
residuals per window) — the batched entries (sdv_ba_set_window_batch, sdv_ba_set_points_batch, sdv_ba_flag_points_batch, sdv_ba_marginalize_points_batch,
sdv_ba_marginalize_frames_batch with the priors out) against the loop of single-window entries (select, set_window, set_points, flag, marginalize points,
marginalize frame, get_prior per window), alternating in one process.  The single-window entries of this library are the n = 1 case of the batched
ones, so the loop arm is this library's n = 1 path (n calls of each), not an earlier release.
  wall ms    host clock around the step (every call ends in a device synchronise); median over the repetitions after one warm-up step
  launches   sdv_launch_count difference over one step
  waits      sdv_ba_host_wait_count difference over one step (optimize_batch included)
  H2D / D2H  bytes the step copies, computed from the shapes: the same rows, header prefixes (8 928 B) and HM/bM for both arms, which differ only in
             the number of copies and in per-call descriptors (a few hundred bytes per window and call); h2d_full_header_path is what single-window
             installs that upload the whole 598 584 B header and the host-built index lists would move, for comparison
Prints the card name, power limit and SM clocks of the same run (not a test).
usage: python tests/_gpu_prof_ba_handover_batch.py [B ...] [--reps R] [--out out.json]"""
import sys, os, json, time, subprocess, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import numpy as np
import sdv_loam_b200  # noqa: F401
from sdv_loam_b200 import api, synth
from conftest import cached_sequence

HDR, PREFIX = 598584, 8928


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("B", nargs="*", type=int, default=[132, 1056]); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out"); a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    seq = cached_sequence(8, 2000, synth.KITTI_K, synth.KITTI_WH); kfs = [0, 1, 2, 3, 4, 5, 6]
    shapes = [synth.make_ba_window(seq, kfs, n_per_frame=243, seed=s, pose_noise=(0.005, 0.0003), match_noise=0.2, prior_scale=1e-3) for s in range(4)]
    nP = int(np.mean([len(w["uv"]) for w in shapes])); nR = int(np.mean([len(w["r_point"]) for w in shapes]))
    print(f"window: {len(kfs)} keyframes, {nP} points, {nR} residuals")
    result = dict(gpu=q, reps=a.reps, points=nP, residuals=nR, runs={})
    ctx = api.Context(synth.KITTI_K, *synth.KITTI_WH, max_frames=len(kfs) + 1, max_kf_images=len(kfs) + 1)
    ids = [500 + k for k in kfs]
    for i, k in enumerate(kfs):
        ctx.makeImages(ids[i], seq.images[k])
    sels = [((w["host"] == 0) | (np.arange(len(w["uv"])) % 4 == 0)).astype(np.int32) * (w["host"] != w["nF"] - 1) for w in shapes]
    for B in a.B:
        W = list(range(B)); wins = [shapes[i % 4] for i in W]; sel = [sels[i % 4] for i in W]

        def batched():                                                       # -> ms of the install and of the hand-over
            t0 = time.perf_counter(); eb = api.EnergyFunctional.install_batch(ctx, W, wins, [ids] * B); t1 = time.perf_counter()
            api.optimize_batch(ctx, W, 6); t2 = time.perf_counter()
            api.flag_points_batch(eb, sel); api.marginalize_points_batch(eb); api.marginalize_frames_batch(eb, [[0]] * B)
            return 1e3 * (t1 - t0 + time.perf_counter() - t2)

        def loop():
            t0 = time.perf_counter(); es = [api.EnergyFunctional(ctx, w, ids, window=k) for k, w in zip(W, wins)]; t1 = time.perf_counter()
            api.optimize_batch(ctx, W, 6); t2 = time.perf_counter()
            for e, s in zip(es, sel):
                e.flagPointsForRemoval(s); e.marginalizePointsF(); e.marginalizeFrame(0); e.prior()
            return 1e3 * (t1 - t0 + time.perf_counter() - t2)

        batched(); loop(); tb, tl = [], []                                   # warm-up, then alternate
        for _ in range(a.reps):
            tb.append(batched()); tl.append(loop())
        l0, w0 = ctx.launch_count(), ctx.ba_host_wait_count(); batched(); lb, wb = ctx.launch_count() - l0, ctx.ba_host_wait_count() - w0
        l0, w0 = ctx.launch_count(), ctx.ba_host_wait_count(); loop(); ll, wl = ctx.launch_count() - l0, ctx.ba_host_wait_count() - w0
        dim = 4 + 6 * len(kfs); d0 = dim - 6
        rows = B * (nP * (96 + 4) + 4 + nR * 28)                             # point and residual rows + the flag selection, both arms
        prior = B * 8 * (d0 * d0 + d0)
        h2d = B * (PREFIX + 8 * (dim * dim + dim)) + rows
        r = dict(batched_ms=float(np.median(tb)), loop_ms=float(np.median(tl)), launches_batched=lb, launches_loop=ll, waits_batched=wb, waits_loop=wl,
                 h2d=h2d, d2h=B * 4 * nP + prior,
                 # whole headers, plus idepth_backup, res_of_target (32 B per point) and the pair lists (4 B per residual + 260 B) built on the host
                 h2d_full_header_path=B * (HDR + nP * (4 + 32) + nR * 4 + 260) + rows)
        print(f"B={B}: install + hand-over (optimize_batch excluded)  batched {r['batched_ms']:.1f} ms  loop of n = 1 calls {r['loop_ms']:.1f} ms  "
              f"launches {lb} vs {ll}  waits {wb} vs {wl}  H2D {h2d/1e6:.1f} MB (full-header path {r['h2d_full_header_path']/1e6:.1f} MB)  D2H {r['d2h']/1e6:.2f} MB")
        result["runs"][B] = r
    ctx.close()
    if a.out:
        json.dump(result, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
