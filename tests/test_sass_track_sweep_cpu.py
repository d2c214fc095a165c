"""The SASS counter of the tracker sweep (tests/_sass_track_sweep.py) still finds what it measures in the built library: one sweep loop per
track_cluster_kernel instantiation, twelve tap gathers (LDGSTS) in it, and no spill traffic inside it."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _sass_track_sweep as sweep  # noqa: E402

LIB = os.path.join(os.path.dirname(HERE), "sdv-loam_b200", "libsdv_b200.so")


@pytest.mark.skipif(not os.path.exists(sweep.CUOBJDUMP), reason="cuobjdump not installed")
def test_one_sweep_loop_per_instantiation():
    assert os.path.exists(LIB), "build() first"
    ks = sweep.kernels(LIB)
    assert set(ks) == {(128, 4), (64, 8), (256, 1)}
    for cfg, loops in ks.items():
        assert len(loops) == 1, (cfg, [(hex(L["lo"]), hex(L["hi"])) for L in loops])
        L = loops[0]
        assert L["ldgsts"] == sweep.TAPS, (cfg, L["ldgsts"])
        assert L["local"] == 0, (cfg, L["local"])
        assert 0 < L["steady"] < L["size"], cfg
