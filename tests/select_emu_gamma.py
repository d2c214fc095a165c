"""ctypes driver of tests/emu/libselect_emu_gamma.so — the REAL kernels + host engine of sdv-loam_b200/csrc/sdv_select_core.cuh compiled for the host (tests/emu/cuda_emu.hpp),
driven with jobs that carry their camera's gamma weights.  TEST INFRASTRUCTURE for tests/test_select_emu_gamma_cpu.py; selector slots come from tests/select_emu.py."""
import ctypes as C
import os
import subprocess
import numpy as np
from select_emu import NEW_TRACE_DTYPE, IMM_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "emu", "libselect_emu_gamma.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        srcs = [os.path.join(_HERE, "emu", "select_emu_gamma.cpp"), os.path.join(_HERE, "emu", "cuda_emu.hpp"), os.path.join(_HERE, "..", "sdv-loam_b200", "csrc", "sdv_select_core.cuh"),
                os.path.join(_HERE, "..", "sdv-loam_b200", "csrc", "sdv_core_common.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-w", "-o", _SO, srcs[0]])
        L = C.CDLL(_SO)
        L.emu_gamma_engine_create.restype = C.c_void_p; L.emu_gamma_engine_create.argtypes = [C.c_int, C.c_int, C.c_void_p]
        L.emu_gamma_engine_destroy.argtypes = [C.c_void_p]; L.emu_gamma_engine_error.restype = C.c_char_p; L.emu_gamma_engine_error.argtypes = [C.c_void_p]
        L.emu_gamma_w2.restype = C.c_float; L.emu_gamma_w2.argtypes = [C.c_float, C.c_void_p]
        L.emu_gamma_make_hists.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.emu_gamma_make_maps.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 14
        L.emu_gamma_make_new_traces.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 14 + [C.c_int] + [C.c_void_p] * 2
        _LIB = L
    return _LIB


def gamma_w2(I, gw2):
    """sdv::gamma_w2 of the device source, compiled for the host"""
    t = None if gw2 is None else np.ascontiguousarray(gw2, np.float32)
    return np.float32(lib().emu_gamma_w2(float(np.float32(I)), None if t is None else t.ctypes.data))


class GammaEngine:
    """the engine fed jobs of several sizes, each with its camera's gamma table gw2 (256 floats) or None"""

    def __init__(self, w, h, rp):
        self.rp = np.ascontiguousarray(rp, np.uint8); self.p = lib().emu_gamma_engine_create(w, h, self.rp.ctypes.data)

    def __del__(self):
        if getattr(self, "p", None):
            lib().emu_gamma_engine_destroy(self.p); self.p = None

    def _ck(self, rc):
        if rc: raise RuntimeError(lib().emu_gamma_engine_error(self.p).decode())

    @staticmethod
    def _tabs(gw2s):
        keep = [None if g is None else np.ascontiguousarray(g, np.float32) for g in gw2s]
        return keep, (C.c_void_p * len(keep))(*[None if g is None else g.ctypes.data for g in keep])

    def makeHists(self, F, wh, gw2):
        n = (wh[0] // 32) * (wh[1] // 32); a = np.zeros(n, np.float32); b = np.zeros(n, np.float32); g = None if gw2 is None else np.ascontiguousarray(gw2, np.float32)
        self._ck(lib().emu_gamma_make_hists(self.p, F.I0.ctypes.data, wh[0], wh[1], None if g is None else g.ctypes.data, a.ctypes.data, b.ctypes.data)); return a, b

    def makeMaps(self, Fs, whs, gw2s, pots, densities, recs, thFactors, clouds=None):
        """one makeMaps / makeMapsFromLidar job per frame -> per-job maps, numHaveSub, final potentials"""
        nj = len(Fs); arr = lambda xs: (C.c_void_p * nj)(*xs); i32 = lambda x: np.ascontiguousarray(x, np.int32); keep, tabs = self._tabs(gw2s)
        w, h = i32([a for a, _ in whs]), i32([b for _, b in whs])
        cl = None if clouds is None else [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]
        sz = [w[j] * h[j] for j in range(nj)] if cl is None else [max(len(c), 1) for c in cl]; off = np.concatenate([[0], np.cumsum(sz)])
        maps = np.zeros(int(off[-1]), np.uint8); pot = i32(pots).copy(); num = np.zeros(nj, np.int32)
        d = np.ascontiguousarray(densities, np.float32); r = i32(recs); t = np.ascontiguousarray(thFactors, np.float32); n = i32([0] * nj if cl is None else [len(c) for c in cl])
        self._ck(lib().emu_gamma_make_maps(self.p, nj, arr([F.I0.ctypes.data for F in Fs]), arr([F.L[0].ctypes.data for F in Fs]), arr([F.L[1].ctypes.data for F in Fs]), tabs,
                                           w.ctypes.data, h.ctypes.data, None if cl is None else arr([c.ctypes.data for c in cl]), n.ctypes.data, d.ctypes.data, r.ctypes.data, t.ctypes.data,
                                           pot.ctypes.data, maps.ctypes.data, num.ctypes.data))
        out = [maps[off[j]:off[j + 1]] for j in range(nj)]
        return ([m.reshape(h[j], w[j]) for j, m in enumerate(out)] if cl is None else [m[:len(c)] for m, c in zip(out, cl)]), num, pot

    def makeNewTraces(self, slots, Fs, whs, gw2s, clouds, densL, densD, add, cap=1 << 14):
        nj = len(slots); cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; arr = lambda xs: (C.c_void_p * nj)(*xs); keep, tabs = self._tabs(gw2s)
        out = np.zeros((nj, cap), NEW_TRACE_DTYPE); imm = np.zeros((nj, cap), IMM_DTYPE); n_out = np.zeros(nj, np.int32); num = np.zeros((nj, 2), np.int32)
        n = np.array([len(c) for c in cl], np.int32); w = np.array([a for a, _ in whs], np.int32); h = np.array([b for _, b in whs], np.int32)
        dl = np.ascontiguousarray(densL, np.float32); dd = np.ascontiguousarray(densD, np.float32); ad = np.ascontiguousarray(add, np.int32)
        self._ck(lib().emu_gamma_make_new_traces(self.p, nj, arr([s.p for s in slots]), arr([F.I0.ctypes.data for F in Fs]), arr([F.L[0].ctypes.data for F in Fs]), arr([F.L[1].ctypes.data for F in Fs]),
                                                 tabs, w.ctypes.data, h.ctypes.data, arr([c.ctypes.data for c in cl]), n.ctypes.data, dl.ctypes.data, dd.ctypes.data, ad.ctypes.data,
                                                 out.ctypes.data, imm.ctypes.data, cap, n_out.ctypes.data, num.ctypes.data))
        return [out[j, :n_out[j]] for j in range(nj)], num
