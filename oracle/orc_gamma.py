"""ctypes binding of oracle/orc_gamma.cpp: frames of a photometrically calibrated camera, and FullSystem::setGammaFunction's inversion.  TEST INFRASTRUCTURE ONLY,
like orc.py, whose liborc.so it links against (oracle/gamma.mk `orc`).  Pinned on the reference's own code by tests/test_ref_pin_gamma.py."""
from __future__ import annotations
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build() -> str:
    """oracle/liborc_gamma.so (make -f gamma.mk orc); in a temporary directory when the tree cannot take it"""
    orc.build()
    try:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "gamma.mk", "orc"])
        return os.path.join(_HERE, "liborc_gamma.so")
    except (subprocess.CalledProcessError, OSError):
        if os.access(_HERE, os.W_OK):
            raise
        d = tempfile.mkdtemp(prefix="orc_gamma_")
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "gamma.mk", "orc", f"OUT={d}"])
        return os.path.join(d, "liborc_gamma.so")


def lib():
    global _LIB
    if _LIB is None:
        orc.lib()                                                     # liborc.so first: the frames are that instance's
        L = C.CDLL(build())
        L.orc_frame_create_gamma.restype = C.c_void_p
        L.orc_frame_create_gamma.argtypes = [orc._f32p, C.c_int, C.c_int, C.c_int, C.c_float, orc._f32p]
        _LIB = L
    return _LIB


def gamma_B(BInv):
    """FullSystem::setGammaFunction (FullSystem.cpp:225-249): CalibHessian::B from BInv (its first 256 values), in the reference's float arithmetic.
    The search runs over s in 1..254 only, an i without a bracket keeps B[i] = i, and B[0] = 0, B[255] = 255."""
    G = np.asarray(BInv, np.float32).reshape(-1)[:256]; f = np.float32
    B = np.arange(256, dtype=f)
    for i in range(1, 255):
        for s in range(1, 255):
            if G[s] <= f(i) and G[s + 1] >= f(i):
                B[i] = f(s) + (f(i) - G[s]) / (G[s + 1] - G[s]); break
    B[0] = 0; B[255] = 255
    return B


class Frame(orc.Frame):
    """orc.Frame after FrameHessian::makeImages with a CalibHessian whose B is set: absSquaredGrad weighed by gw^2; B None: the identity (orc.Frame itself)"""

    def __init__(self, color, levels: int, exposure: float = 1.0, B=None):
        if B is None:
            super().__init__(color, levels, exposure); return
        color = np.ascontiguousarray(color, np.float32)
        self.h, self.w = color.shape
        self.levels = levels
        self.p = lib().orc_frame_create_gamma(color, self.w, self.h, levels, exposure, np.ascontiguousarray(B, np.float32).reshape(256))
