"""GPU (-m gpu) counterpart of tests/test_sequence_distmap.py: CoarseDistanceMap::makeDistanceMap and the activation walk of activatePointsMT on the device, for the
18 LIVE windows of the reference's own run (tests/golden/seq_distmap_ref.npz: 930 - 1 310 forward-warped source points per window, real poses, bundle-adjusted K), all
18 as sequences of ONE activateSelectBatch call, against the reference's stored digests of the map before the walk, the decisions and the map after it.  The candidates
are the ones test_sequence_distmap.py draws, from the same generator stream in window order.  On a mismatch the first differing pixel or candidate is reported
against the oracle (orc.DistMap)."""
import numpy as np
import pytest
import orc
from ref_golden import _digest
from test_sequence_distmap import GOLD, _candidates

pytestmark = pytest.mark.gpu


def _sequences(g, w, h):
    """per window: the sources (every keyframe but the newest, grouped by host), the candidates on every keyframe, and the minimum activation distance"""
    rng = np.random.default_rng(11); out = []
    for i in g["windows"]:
        p = f"w{i}_"; KRKi, Kt, host = g[p + "KRKi"], g[p + "Kt"], g[p + "host"].astype(np.int32); nF = len(KRKi)
        p3 = np.concatenate([g[p + "uv"].astype(np.float32), g[p + "idepth"][:, None]], 1)
        hosts = [k for k in range(nF) if k != nF - 1]
        uvid = [p3[host == k] for k in hosts]; pb = np.concatenate([[0], np.cumsum([len(u) for u in uvid])]).astype(np.int32)
        cand, cb, minDist = _candidates(rng, nF, w, h)
        out.append(dict(pt_begin=pb, KRKi=KRKi[hosts], Kt=Kt[hosts], uvid=np.concatenate(uvid).astype(np.float32),
                        cand_begin=np.asarray(cb, np.int32), cKRKi=KRKi, cKt=Kt, cand4=cand, minActDist=minDist))
    return out


def _first_diff(a, b):
    a, b = np.asarray(a), np.asarray(b); eq = (a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else a == b
    k = np.unravel_index(int(np.argmin(eq)), a.shape)
    return k, a[k], b[k]


def test_live_windows_in_one_batch():
    import sdv_loam_b200  # noqa: F401
    from sdv_loam_b200 import api, synth
    w, h = synth.KITTI_WH; g = np.load(GOLD); seqs = _sequences(g, w, h); n = len(seqs)
    assert n == 18
    ctx = api.Context(synth.KITTI_K, w, h)
    api.PixelSelector(ctx, 1, api.random_pattern(w, h))
    _, before = api.activateSelectBatch(ctx, [{k: q[k] for k in ("pt_begin", "KRKi", "Kt", "uvid")} for q in seqs], want_maps=True)
    decs, after = api.activateSelectBatch(ctx, seqs, want_maps=True)
    accepted = 0
    for j, (i, q) in enumerate(zip(g["windows"], seqs)):
        p = f"w{i}_"; od = None
        for what, got, key in (("map", before[j], "map"), ("decisions", decs[j], "decisions"), ("map after the walk", after[j], "map_after")):
            if _digest(got) == g[p + key].item():
                continue
            od = orc.DistMap(w >> 1, h >> 1); od.make(q["pt_begin"], q["KRKi"], q["Kt"], q["uvid"]); om = od.get().copy()
            od_dec = od.activateSelect(q["cand_begin"], q["cKRKi"], q["cKt"], q["cand4"], q["minActDist"])
            want = {"map": om, "decisions": od_dec, "map_after": od.get()}[key]
            k, a, b = _first_diff(got, want)
            raise AssertionError(f"window {i} {what}: differs from the reference's digest; first difference from the oracle at {k}: device {a!r}, oracle {b!r}")
        accepted += int((decs[j] == 1).sum())
    assert accepted > 500, accepted
    for j in range(n):                                                       # per-window calls equal the batched call
        d1, m1 = api.activateSelectBatch(ctx, [seqs[j]], want_maps=True)
        assert np.array_equal(d1[0], decs[j]) and np.array_equal(m1[0], after[j], equal_nan=True), j
    ctx.close()
