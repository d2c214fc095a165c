"""ctypes binding of oracle/ref_gamma_shim.cpp and oracle/ref_photo_shim.cpp: the reference's own code for a photometrically calibrated camera — its
PhotometricUndistorter (constructor, getG, processFrame), FullSystem::setGammaFunction and FrameHessian::makeImages with that CalibHessian.  TEST INFRASTRUCTURE
ONLY; needs oracle/_ref (built where the reference sources are present), so only the recording of tests/golden/ref_pin_gamma.npz loads it."""
from __future__ import annotations
import ctypes as C
import os
import subprocess

import numpy as np
import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_PHOTO = None
_f32p, _vp = ref._f32p, ref._vp


def _build():
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "gamma.mk", "ref", f"REF={ref.REF_SRC}"])


def lib():
    global _LIB
    if _LIB is None:
        ref.lib()                                                     # libsdvref.so first: the shim works on the objects of that instance
        _build()
        L = C.CDLL(os.path.join(_HERE, "_ref", "libsdvref_gamma.so"), mode=os.RTLD_NOW)
        L.ref_gamma_set.argtypes = [_vp, _vp, _f32p]; L.ref_gamma_set.restype = None
        L.ref_gamma_make_images.argtypes = [_vp, _vp, _f32p]; L.ref_gamma_make_images.restype = None
        _LIB = L
    return _LIB


def photo_lib():
    global _PHOTO
    if _PHOTO is None:
        _build()
        L = C.CDLL(os.path.join(_HERE, "_ref", "libsdvref_photo.so"), mode=os.RTLD_NOW)
        L.ref_photo_create.restype = _vp; L.ref_photo_create.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
        L.ref_photo_destroy.argtypes = [_vp]; L.ref_photo_destroy.restype = None
        L.ref_photo_get.argtypes = [_vp, C.POINTER(C.c_int), _vp, _vp]
        L.ref_photo_process.argtypes = [_vp, _vp, C.c_float, C.c_float, C.c_int, _f32p]; L.ref_photo_process.restype = None
        _PHOTO = L
    return _PHOTO


def set_gamma(S, G) -> np.ndarray:
    """FullSystem::setGammaFunction(G) on ref.System S (G None: a NULL pointer) -> CalibHessian::B"""
    B = np.zeros(256, np.float32); g = None if G is None else np.ascontiguousarray(G, np.float32)
    lib().ref_gamma_set(S.p, None if g is None else g.ctypes.data, B); return B


def make_images(S, frame, color):
    """FrameHessian::makeImages(color, &S.Hcalib) on a ref.Frame: its absSquaredGrad is then weighed with S's gamma"""
    with ref._Quiet():
        lib().ref_gamma_make_images(S.p, frame.p, np.ascontiguousarray(color, np.float32).reshape(-1))


class Photometric:
    """the reference's PhotometricUndistorter(gamma_file, "", vignette_file, w, h) with setting_photometricCalibration = pc"""

    def __init__(self, gamma_file, vignette_file, w, h, pc=2):
        self.w, self.h, self.pc = w, h, pc; L = photo_lib()
        with ref._Quiet():
            self.p = L.ref_photo_create((gamma_file or "").encode(), (vignette_file or "").encode(), w, h, pc)

    def state(self):
        """(valid, GDepth, getG() or None, vignetteMapInv or None)"""
        L = photo_lib(); gd = C.c_int(0); L.ref_photo_get(self.p, C.byref(gd), None, None)
        G = np.zeros(max(gd.value, 1), np.float32); V = np.full(self.w * self.h, np.nan, np.float32)
        valid = L.ref_photo_get(self.p, C.byref(gd), G.ctypes.data, V.ctypes.data)
        return bool(valid), gd.value, (G[:gd.value] if valid else None), (None if np.isnan(V).all() else V.reshape(self.h, self.w))

    def processFrame(self, raw, exposure=1.0, factor=1.0):
        out = np.zeros(self.w * self.h, np.float32); r = np.ascontiguousarray(raw, np.uint8)
        photo_lib().ref_photo_process(self.p, r.ctypes.data, exposure, factor, self.pc, out); return out.reshape(self.h, self.w)

    def __del__(self):
        if getattr(self, "p", None) and _PHOTO is not None:
            _PHOTO.ref_photo_destroy(self.p); self.p = None
