"""The float64 tracker reference (tests/tracker_fp64.py) against the oracle's calcRes / calcGSSSE, on the CPU.

The oracle is pinned bit for bit to the reference implementation; it sums E and the flow indicators in one float and H/b in four SSE lanes
with 1000-term tiers.  The float64 reference must agree with it on nE and nSat exactly and on E, H, b and the flow indicators within the
oracle's own float-summation bound.  That is what lets the GPU tests treat the reference as ground truth."""
import numpy as np
import orc
import tracker_fp64 as tf
from conftest import SMALL_K, SMALL_WH

ID7 = np.array([1, 0, 0, 0, 0, 0, 0.0])


def _setup(seq, K, wh, n):
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import synth
    w, h = wh; L = 4
    pts = synth.select_points(seq.images[0], seq.clouds[0], n)
    p4 = np.concatenate([pts, np.full((len(pts), 1), 1e-3, np.float32)], 1).astype(np.float32)
    f0, f1 = orc.Frame(seq.images[0], L), orc.Frame(seq.images[1], L)
    otr = orc.CoarseTracker(w, h, L, K); otr.setCoarseTrackingRef(f0, p4, np.zeros(len(p4), np.int32), 0.0, 1.0)
    Tgt = orc.se3_from_rt(*synth.rel_pose(seq.R[0], seq.t[0], seq.R[1], seq.t[1]))
    poses = {"identity": ID7, "near": orc.se3_mul(orc.se3_exp([0.01, 0.0, 0.02, 1e-3, -1e-3, 5e-4]), Tgt),
             "far": orc.se3_exp([0.3, -0.1, 0.5, 0.02, 0.03, -0.01])}
    return otr, f0, f1, L, poses


def _check_against_oracle(otr, f1, lvl, T, a, b, cutoff, rep, tag, ref_b=1.0):
    ref = tf.Ref(otr, f1, lvl, T, a, b, cutoff, ref_b=ref_b)
    ro = ref.rs_oracle
    assert int(ro[1]) == ref.nE
    mE = ref.nE                                                    # one float, every term in sequence
    mF = max(1, ref.n_flow // 2)                                   # sum_bound doubles m for the flow entries
    rep.check(tag + " E", abs(ro[0] - ref.rs[0]), ref.sum_bound(tf.IDX_E, mE))
    fN = float(np.float32(ref.n_flow)) + 0.1
    rep.check(tag + " flowT", abs(ro[2] - ref.rs[2]), ref.sum_bound(tf.IDX_FT, mF) / fN)
    rep.check(tag + " flowRT", abs(ro[4] - ref.rs[4]), ref.sum_bound(tf.IDX_FRT, mF) / fN)
    Ho, bo = otr.calcGSSSE(lvl, T, a, b)
    ref.check_gs(Ho, bo, tf.m_oracle_gs(ref.npad), rep, tag)
    return ref


def test_reference_matches_oracle(small_seq, kitti_seq):
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import synth
    rep = tf.Report("fp64 reference vs oracle"); residues = set()
    for name, seq, K, wh, n in (("small", small_seq, SMALL_K, SMALL_WH, 800), ("kitti", kitti_seq, synth.KITTI_K, synth.KITTI_WH, 2000)):
        otr, f0, f1, L, poses = _setup(seq, K, wh, n)
        for pname, T in poses.items():
            for lvl in range(L):
                for cutoff, (a, b) in ((20.0, (0.0, 0.0)), (40.0, (0.03, -2.0))):
                    ref = _check_against_oracle(otr, f1, lvl, T, a, b, cutoff, rep, f"{name}")
                    if ref.nW:
                        residues.add(ref.nW % 4)
        # every residue of the warped count mod 4 (the npad rule): the level-0 cloud cut to n, n-1, n-2, n-3 points
        cu = otr.cloud(0)
        for d in range(4):
            k = len(cu[0]) - d
            otr.setCloud(f0, 0, *(c[:k] for c in cu), 0.0, 1.0)
            ref = _check_against_oracle(otr, f1, 0, poses["near"], 0.0, 0.0, 20.0, rep, f"{name} cut")
            residues.add(ref.nW % 4)
    rep.print()
    assert residues == {0, 1, 2, 3}, residues


def test_bound_geometry():
    """m from the launch geometry: the step-wise grid cap and the LM stride."""
    assert tf.m_step(0, 132) == 0 and tf.m_step(1, 132) == 1 and tf.m_step(4 * 132 * 256, 132) == 1 and tf.m_step(4 * 132 * 256 + 1, 132) == 2
    assert tf.m_step(163840, 132) == 2
    assert tf.m_lm(163840, 128, 1) == 1280 and tf.m_lm(4096, 256, 16) == 1 and tf.m_lm(4097, 256, 16) == 2
