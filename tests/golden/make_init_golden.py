"""Writes tests/golden/seq_init_ref.npz from the REFERENCE's own code (oracle/_ref + oracle/ref_init_shim.cpp, built where the reference sources are present).
Run from the repo root:  python tests/golden/make_init_golden.py

  seq_init_ref.npz   the reference's FullSystem over the first two frames of S-KITTI-200 with srand(seed) before frame 1: frame 0's pixel rows and box, the seed,
                     numPoints[0], and frame 1's camToTrackingRef, aff_g2l and lastCoarseRMSE                                     (tests/test_gpu_init.py)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
INIT_SEED = 20261017


def main():
    """the start of a sequence in the reference's own FullSystem: frame 0 (setFirstFromLidar) and frame 1 (initializeFromInitializer, setCTRefForFirstFrame, the
    53-hypothesis trackNewCoarse), with the LiDAR box the node would have set (main.cpp:833-836) and srand(INIT_SEED) right before frame 1"""
    import ref
    import ref_init
    import seq_replay as sr
    from test_sequence_parity import _seq
    seq, synth = _seq(); w, h = seq.wh
    L = ref.set_calib(w, h, seq.K)
    S = ref.System(L, perfect_images=True)
    box = np.array([10000, -1, 10000, -1], np.int32); clouds = []
    for i in range(2):
        cl = sr.frame_cloud(seq, i); clouds.append(cl)
        box = np.array([min(box[0], int(cl[:, 0].min())), max(box[1], int(cl[:, 0].max())), min(box[2], int(cl[:, 1].min())), max(box[3], int(cl[:, 1].max()))], np.int32)
        S.set_lidar_state(box, 1)
        if i == 0:
            box0 = box.copy()
        else:
            S.srand(INIT_SEED)
        assert S.addActiveFrame(seq.images[i], cl, 0.1 * i) == 0, i
        if i == 0:
            n_sel = ref_init.init_num_points(S)
    r = S.frame(1)
    np.savez_compressed(os.path.join(HERE, "seq_init_ref.npz"), rows0=clouds[0], lrud0=box0, seed=np.int64(INIT_SEED), levels=np.int32(L), n_selected=np.int32(n_sel),
                        camToTrackingRef=r["camToTrackingRef"], aff_g2l=r["aff_g2l"], lastCoarseRMSE=S.lastCoarseRMSE())


if __name__ == "__main__":
    main()
