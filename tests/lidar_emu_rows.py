"""ctypes driver of tests/emu/liblidar_emu_rows.so — the LiDAR front-end of sdv-loam_b200/csrc/sdv_lidar_core.cuh compiled for the host (tests/emu/cuda_emu.hpp) and driven
through its device-output path: rows into row-set blocks, the running pixel box kept in "device" memory between calls, one header per sweep.
TEST INFRASTRUCTURE for tests/test_lidar_emu_rows_cpu.py."""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "emu", "liblidar_emu_rows.so")
_LIB = None
HDR_FIELDS = ["rows", "overflow", "left", "right", "up", "down", "addFeaturePoint", "numGround", "n_segmented"]
HDR_DTYPE = np.dtype([(f, np.int32) for f in HDR_FIELDS] + [("pad", np.int32, 7)])


def lib():
    global _LIB
    if _LIB is None:
        srcs = [os.path.join(_HERE, "emu", "lidar_emu_rows.cpp"), os.path.join(_HERE, "emu", "cuda_emu.hpp"), os.path.join(_HERE, "..", "sdv-loam_b200", "csrc", "sdv_lidar_core.cuh"),
                os.path.join(_HERE, "..", "sdv-loam_b200", "csrc", "sdv_core_common.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-w", "-o", _SO, srcs[0]])
        L = C.CDLL(_SO)
        L.emu_rows_create.restype = C.c_void_p; L.emu_rows_create.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]
        L.emu_rows_destroy.argtypes = [C.c_void_p]; L.emu_rows_error.restype = C.c_char_p; L.emu_rows_error.argtypes = [C.c_void_p]
        L.emu_rows_handle.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p]
        assert L.emu_rows_header_bytes() == HDR_DTYPE.itemsize
        _LIB = L
    return _LIB


class RowsEngine:
    """the handler with its state the way the library keeps it: one box per selector slot, one row-set block (header + room for cap rows) per frame"""

    def __init__(self, n_slots, n_scan=64, horizon=1800, ang_res_x=0.2, ang_res_y=0.427, ang_bottom=24.9, groundScanInd=50):
        self.p = lib().emu_rows_create(n_scan, horizon, ang_res_x, ang_res_y, ang_bottom, groundScanInd)
        self.boxes = np.tile(np.array([10000, -1, 10000, -1], np.int32), (n_slots, 1))     # FullSystem::left/right/up/down per slot, their initial values
        self.sets = {}

    def __del__(self):
        if getattr(self, "p", None):
            lib().emu_rows_destroy(self.p); self.p = None

    def handle(self, slots, frames, sweeps, Rlc, tlc, K4, wh, cap, stats=False, slack=64):
        """sweep j of the sequence on slots[j] into frames[j]'s set (cap rows of room; `slack` rows past it hold a NaN sentinel) -> stats (nj, 5) or None"""
        nj = len(slots); sw = [np.ascontiguousarray(s, np.float32).reshape(-1, 4) for s in sweeps]
        allp = np.ascontiguousarray(np.concatenate(sw)) if nj else np.zeros((0, 4), np.float32); offs = np.concatenate([[0], np.cumsum([len(s) for s in sw])])
        ptrs = (C.c_void_p * nj)(*[allp.ctypes.data + 16 * int(offs[j]) for j in range(nj)]); n = np.array([len(s) for s in sw], np.int32)
        box = np.ascontiguousarray(self.boxes[slots]); blocks = np.full((nj, cap + slack, 3), np.nan); hdr = np.zeros(nj, HDR_DTYPE)
        R = np.ascontiguousarray(Rlc, np.float64).reshape(-1); t = np.ascontiguousarray(tlc, np.float64); K = np.ascontiguousarray(K4, np.float32); st = np.zeros((nj, 5), np.int32) if stats else None
        rc = lib().emu_rows_handle(self.p, nj, ptrs, n.ctypes.data, R.ctypes.data, t.ctypes.data, K.ctypes.data, wh[0], wh[1], box.ctypes.data, blocks.ctypes.data, (cap + slack) * 3,
                                   hdr.ctypes.data, cap, None if st is None else st.ctypes.data)
        if rc: raise RuntimeError(lib().emu_rows_error(self.p).decode())
        self.boxes[slots] = box
        for j, f in enumerate(frames):
            self.sets[f] = dict(hdr=hdr[j], block=blocks[j], cap=cap)
        return st
