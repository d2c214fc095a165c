"""ctypes binding of oracle/orc_init.cpp: the restatement of the start of a sequence (CoarseInitializer::setFirstFromLidar at level 0, the point loop of
FullSystem::initializeFromInitializer, setCTRefForFirstFrame).  TEST INFRASTRUCTURE ONLY, like orc.py, whose liborc.so it links against (oracle/init.mk).
Pinned on the reference's own code by tests/test_ref_pin_init.py."""
from __future__ import annotations
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
INIT_META_DTYPE = np.dtype([("my_type", "<f4"), ("type", "<i4"), ("isFromSensor", "<i4"), ("idepth_fromSensor", "<f4")])   # sdv_immature_meta


def build() -> str:
    """oracle/liborc_init.so (make -f init.mk orc); in a temporary directory when the tree cannot take it"""
    orc.build()
    try:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "init.mk", "orc"])
        return os.path.join(_HERE, "liborc_init.so")
    except (subprocess.CalledProcessError, OSError):
        if os.access(_HERE, os.W_OK):
            raise
        d = tempfile.mkdtemp(prefix="orc_init_")
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "init.mk", "orc", f"OUT={d}"])
        return os.path.join(d, "liborc_init.so")


def lib():
    global _LIB
    if _LIB is None:
        orc.lib()                                                     # liborc.so first: the restatement resolves its pieces in that instance
        L = C.CDLL(build())
        L.orc_init_from_lidar.restype = C.c_int
        L.orc_init_from_lidar.argtypes = [C.c_void_p, C.c_int, C.c_int, orc._u8p, C.c_void_p, C.c_int, orc._i32p, C.c_float, orc._i32p, C.c_void_p, orc._i32p, orc._f32p,
                                          orc._i32p, C.c_void_p, C.c_void_p, orc._f32p]
        _LIB = L
    return _LIB


def init_from_lidar(frame, random_pattern, cloud3, lrud, desiredPointDensity, draws, tracker=None):
    """CoarseInitializer::setFirstFromLidar (level 0) + the point loop of FullSystem::initializeFromInitializer on `frame` (an orc.Frame), and setCTRefForFirstFrame
    into `tracker` (an orc.CoarseTracker, optional).  random_pattern: at least w*h bytes; draws: rand() values, at least one per row.
    -> dict(n_selected, pnt (n_selected, 5) {u, v, my_type, mdepth, isFromSensor}, keep (n_selected,), pts orc.IMM_DTYPE, meta INIT_META_DTYPE, idepth)"""
    L = lib(); w, h = frame.w, frame.h
    c = np.ascontiguousarray(cloud3, np.float64).reshape(-1, 3); n = len(c); m = max(n, 1)
    d = np.ascontiguousarray(draws, np.int32); assert len(d) >= n
    rp = np.ascontiguousarray(np.asarray(random_pattern, np.uint8).reshape(-1)[:w * h])
    nsel = np.zeros(1, np.int32); pnt = np.zeros((m, 5), np.float32); keep = np.zeros(m, np.int32)
    pts = np.zeros(m, orc.IMM_DTYPE); meta = np.zeros(m, INIT_META_DTYPE); idp = np.zeros(m, np.float32)
    k = L.orc_init_from_lidar(frame.p, w, h, rp, c.ctypes.data if n else None, n, np.ascontiguousarray(lrud, np.int32), desiredPointDensity, d if len(d) else np.zeros(1, np.int32),
                              None if tracker is None else tracker.p, nsel, pnt.reshape(-1), keep, pts.ctypes.data, meta.ctypes.data, idp)
    if tracker is not None:
        tracker._ref = frame
    ns = int(nsel[0])
    return dict(n_selected=ns, pnt=pnt[:ns].copy(), keep=keep[:ns].copy(), pts=pts[:k].copy(), meta=meta[:k].copy(), idepth=idp[:k].copy())
