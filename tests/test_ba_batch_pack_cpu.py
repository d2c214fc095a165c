"""api.pack_ba_windows (the concatenation behind EnergyFunctional.install_batch) against hand-built concatenations: windows with zero points, with zero
residuals and of one frame, value_zero and priors given for some windows only."""
import numpy as np


def _win(rng, nF, nP, per_point, prior=False, kzero=False):
    host = np.sort(rng.integers(0, nF, nP)).astype(np.int32)
    rb = [0]; rp, rh, rt = [], [], []
    for p in range(nP):
        tg = [t for t in range(nF) if t != host[p]][:per_point]
        for t in tg:
            rp.append(p); rh.append(host[p]); rt.append(t)
        rb.append(len(rp))
    nR = len(rp); d = 4 + 6 * nF
    w = dict(nF=nF, K=rng.normal(size=4) + 600, T_eval=rng.normal(size=(nF, 7)), state=rng.normal(size=(nF, 10)), state_zero=rng.normal(size=(nF, 10)),
             ab_exposure=rng.random(nF).astype(np.float32), frameID=np.arange(nF, dtype=np.int32), frameEnergyTH=rng.random(nF).astype(np.float32),
             uv=rng.random((nP, 2)).astype(np.float32), idepth=rng.random(nP).astype(np.float32), idepth_zero=rng.random(nP).astype(np.float32),
             color=rng.random((nP, 8)).astype(np.float32), weights=rng.random((nP, 8)).astype(np.float32), host=host,
             hasDepthPrior=rng.integers(0, 2, nP).astype(np.int32), isFromSensor=rng.integers(0, 2, nP).astype(np.int32), res_begin=np.array(rb, np.int32),
             r_point=np.array(rp, np.int32), r_host=np.array(rh, np.int32), r_target=np.array(rt, np.int32), r_hasMatcher=np.ones(nR, np.int32),
             r_matcher=rng.random((nR, 2)).astype(np.float32), r_isNew=np.zeros(nR, np.int32))
    if prior:
        w["HM"] = rng.normal(size=(d, d)); w["bM"] = rng.normal(size=d)
    if kzero:
        w["K_zero"] = rng.normal(size=4)
    return w


def test_pack_matches_hand_concatenation():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api
    rng = np.random.default_rng(5)
    wins = [_win(rng, 4, 30, 2, prior=True), _win(rng, 3, 0, 0), _win(rng, 5, 12, 0, kzero=True), _win(rng, 1, 7, 0), _win(rng, 8, 40, 7, prior=True)]
    ids = [list(range(100 * i, 100 * i + w["nF"])) for i, w in enumerate(wins)]
    k = api.pack_ba_windows(wins, ids)
    assert k["n"] == 5
    assert list(k["f_begin"]) == [0, 4, 7, 12, 13, 21]
    assert list(k["p_begin"]) == [0, 30, 30, 42, 49, 89]
    nR = [len(w["r_point"]) for w in wins]
    assert nR[1] == nR[2] == nR[3] == 0 and list(k["r_begin"]) == list(np.concatenate([[0], np.cumsum(nR)]))
    assert k["frame_ids"].dtype == np.uint64 and list(k["frame_ids"]) == sum(ids, [])
    for key, t in (("T_eval", np.float64), ("state", np.float64), ("uv", np.float32), ("color", np.float32), ("host", np.int32), ("r_target", np.int32),
                   ("r_matcher", np.float32), ("frameEnergyTH", np.float32)):
        want = np.concatenate([np.asarray(w[key], t).reshape(-1) for w in wins])
        assert k[key].dtype == t and np.array_equal(k[key], want), key
    # res_begin: window i's block of nP_i + 1 entries starts at p_begin[i] + i, window-local
    assert len(k["res_begin"]) == 89 + 5
    for i, w in enumerate(wins):
        s = k["p_begin"][i] + i
        assert np.array_equal(k["res_begin"][s:s + len(w["uv"]) + 1], w["res_begin"])
    assert np.array_equal(k["K"], np.concatenate([w["K"] for w in wins]))
    sf = np.float64(np.float32(1) / np.float32(50))                         # value_zero = value for the windows without one
    want = np.concatenate([w["K_zero"] if "K_zero" in w else w["K"] * sf for w in wins])
    assert np.array_equal(k["K_zero"], want)
    dims = [4 + 6 * w["nF"] for w in wins]
    hm = np.concatenate([(w["HM"] if "HM" in w else np.zeros((d, d))).reshape(-1) for w, d in zip(wins, dims)])
    bm = np.concatenate([w["bM"] if "bM" in w else np.zeros(d) for w, d in zip(wins, dims)])
    assert np.array_equal(k["HM"], hm) and np.array_equal(k["bM"], bm)


def test_pack_without_prior_or_value_zero():
    import sdv_loam_b200  # noqa
    from sdv_loam_b200 import api
    rng = np.random.default_rng(6)
    wins = [_win(rng, 2, 5, 1), _win(rng, 1, 0, 0)]
    k = api.pack_ba_windows(wins, [[1, 2], [3]])
    assert k["K_zero"] is None and k["HM"] is None and k["bM"] is None
    assert list(k["p_begin"]) == [0, 5, 5] and list(k["res_begin"]) == list(wins[0]["res_begin"]) + [0]
