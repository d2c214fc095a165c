"""ctypes binding of oracle/ref_init_shim.cpp: the reference's own members of the start of a sequence, one at a time, on a ref.System and ref.Frames
(setFirstFromLidar, initializeFromInitializer, setCTRefForFirstFrame).  TEST INFRASTRUCTURE ONLY; needs oracle/_ref (built where the reference sources are present),
so only the recording of tests/golden/ref_pin_init.npz and seq_init_ref.npz loads it."""
from __future__ import annotations
import ctypes as C
import os
import subprocess

import numpy as np
import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_f32p, _f64p, _i32p, _vp = ref._f32p, ref._f64p, ref._i32p, ref._vp


def lib():
    global _LIB
    if _LIB is None:
        ref.lib()                                                     # libsdvref.so first: the shim works on the objects of that instance
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "init.mk", "ref", f"REF={ref.REF_SRC}"])
        L = C.CDLL(os.path.join(_HERE, "_ref", "libsdvref_init.so"), mode=os.RTLD_NOW)
        L.ref_init_first.argtypes = [_vp, _vp, _f64p, C.c_int, _i32p, _f32p]
        L.ref_init_from_initializer.argtypes = [_vp, _vp, C.c_uint, C.c_float, _f32p, C.c_int]
        L.ref_init_num_points.argtypes = [_vp]
        L.ref_init_tracker_set_first.argtypes = [_vp, _vp]; L.ref_init_tracker_set_first.restype = None
        _LIB = L
    return _LIB


def init_first(S, frame, cloud_px, lrud):
    """CoarseInitializer::setFirstFromLidar of ref.System S on frame (a ref.Frame) -> Pnt list of level 0 (numPoints[0], 5) {u, v, my_type, mdepth, isFromSensor}"""
    cl = np.ascontiguousarray(cloud_px, np.float64).reshape(-1, 3); o = np.zeros((max(len(cl), 1), 5), np.float32)
    S._first = frame
    with ref._Quiet():
        m = lib().ref_init_first(S.p, frame.p, cl if len(cl) else np.zeros((1, 3)), len(cl), np.ascontiguousarray(lrud, np.int32), o.reshape(-1))
    return o[:m].copy()


def init_from_initializer(S, new_frame, seed, desiredPointDensity, cap=1 << 16):
    """setting_desiredPointDensity = desiredPointDensity; srand(seed); FullSystem::initializeFromInitializer(new_frame); HdiF = 0
    -> (n, 26) float32 PointHessian rows of the first frame (see ref_init_shim.cpp)"""
    o = np.zeros((cap, 26), np.float32); S._second = new_frame
    with ref._Quiet():
        m = lib().ref_init_from_initializer(S.p, new_frame.p, seed, desiredPointDensity, o.reshape(-1), cap)
    return o[:m].copy()


def init_num_points(S) -> int:
    """CoarseInitializer::numPoints[0] of S's last setFirstFromLidar"""
    return int(lib().ref_init_num_points(S.p))


def tracker_set_first(S, tracker):
    """CoarseTracker::setCTRefForFirstFrame(frameHessians) of S into a ref.CoarseTracker"""
    lib().ref_init_tracker_set_first(S.p, tracker.p); tracker._keep = (S._first, None)
