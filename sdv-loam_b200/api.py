"""ctypes host mirror of the reference call surface over libsdv_b200.so (include/sdv_b200.h).

Classes keep the reference's member names and argument meaning so parity tests read like calls into the original:
  Context                      one FullSystem's device state (sdv_create/sdv_destroy)
  Context.makeImages           FrameHessian::makeImages            src/FullSystem/HessianBlocks.cpp:107-167
  CoarseTracker.setCoarseTrackingRef / calcRes / calcGSSSE / trackNewestCoarse
                               src/FullSystem/CoarseTracker.cpp:649-660, 486-634, 427-484, 662-838
There is no CPU fallback: if the library cannot be loaded this module raises at import time.
"""
from __future__ import annotations
import ctypes as C
import os
import numpy as np
from .build import library_path

PYR_LEVELS = 6


class sdv_calib(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class sdv_settings(C.Structure):
    _fields_ = [("huberTH", C.c_float), ("coarseCutoffTH", C.c_float), ("affineOptModeA", C.c_float), ("affineOptModeB", C.c_float),
                ("outlierTH", C.c_float), ("outlierTHSumComponent", C.c_float), ("idepthFixPrior", C.c_float),
                ("max_ref_points", C.c_int), ("n_tracker_slots", C.c_int), ("max_frames", C.c_int), ("cluster_size", C.c_int),
                ("track_threads", C.c_int), ("max_kf_images", C.c_int)]


class sdv_track_stats(C.Structure):
    _fields_ = [("point_evals", C.c_int64 * PYR_LEVELS), ("iterations", C.c_int32 * PYR_LEVELS), ("accepts", C.c_int32 * PYR_LEVELS)]


MAP_PT_DTYPE = np.dtype([("u", np.float32), ("v", np.float32), ("idepth", np.float32), ("host", np.int32), ("type", np.int32)])
OVERLAP_PT_DTYPE = np.dtype([("u", np.float32), ("v", np.float32), ("idepth", np.float32), ("host", np.int32), ("obs_x", np.float32), ("obs_y", np.float32)])
TRACK_STATS_DTYPE = np.dtype([("point_evals", np.int64, PYR_LEVELS), ("iterations", np.int32, PYR_LEVELS), ("accepts", np.int32, PYR_LEVELS)])
assert TRACK_STATS_DTYPE.itemsize == C.sizeof(sdv_track_stats)

_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")
_vp = C.c_void_p


def _load():
    path = library_path()
    if not os.path.exists(path):
        raise ImportError(f"{path} is not built: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
    L = C.CDLL(path)
    L.sdv_default_settings.argtypes = [C.POINTER(sdv_settings)]
    L.sdv_create.argtypes = [C.POINTER(sdv_calib), C.c_int, C.c_int, C.c_int, C.POINTER(sdv_settings), C.c_int, C.POINTER(_vp)]
    L.sdv_destroy.argtypes = [_vp]; L.sdv_destroy.restype = None
    L.sdv_last_error.argtypes = [_vp]; L.sdv_last_error.restype = C.c_char_p
    L.sdv_pyr_levels.argtypes = [C.c_int, C.c_int]
    L.sdv_sync.argtypes = [_vp]
    L.sdv_set_calib.argtypes = [_vp, C.POINTER(sdv_calib)]
    L.sdv_set_calib_slots.argtypes = [_vp, C.c_int, _i32p, _vp]
    L.sdv_set_calib_slots_cams.argtypes = [_vp, C.c_int, _i32p, _vp, _vp]
    L.sdv_set_camera_size.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.sdv_set_camera_levels.argtypes = [_vp, C.c_int, C.c_int]
    L.sdv_set_camera_storage.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.sdv_camera_storage_bytes.argtypes = [_vp, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.sdv_frame_upload_batch_cams.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _vp, C.c_int, _f32p]
    L.sdv_frame_build_batch_dev_cams.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _vp, C.c_int, _f32p]
    L.sdv_frame_upload.argtypes = [_vp, C.c_uint64, _vp, C.c_float]
    L.sdv_frame_upload_batch.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _f32p]
    L.sdv_frame_upload_batch_u8.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _f32p]
    L.sdv_frame_build_batch_dev.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), C.c_int, _f32p]
    L.sdv_set_undistort.argtypes = [_vp, C.c_int, C.c_int, _f32p, _f32p, C.c_float, _vp, _vp]
    L.sdv_frame_upload_batch_raw_u8.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _f32p]
    L.sdv_set_undistort_cam.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _f32p, _f32p, C.c_float, _vp, _vp]
    L.sdv_frame_upload_batch_raw_u8_cams.argtypes = [_vp, C.c_int, _u64p, C.POINTER(_vp), _vp, _f32p]
    L.sdv_set_gamma_cam.argtypes = [_vp, C.c_int, _vp]
    L.sdv_track_job_bytes.argtypes = []
    L.sdv_launch_count.argtypes = [_vp]; L.sdv_launch_count.restype = C.c_longlong
    L.sdv_frame_release.argtypes = [_vp, C.c_uint64]
    L.sdv_frame_download.argtypes = [_vp, C.c_uint64, C.c_int, _vp, _vp]
    L.sdv_tracker_set_ref.argtypes = [_vp, C.c_int, C.c_uint64, C.c_int, _f32p, _i32p, C.c_float, C.c_double, C.c_double]
    L.sdv_tracker_set_cloud.argtypes = [_vp, C.c_int, C.c_uint64, C.c_int, C.c_int, _f32p, _f32p, _f32p, _f32p, C.c_double, C.c_double]
    L.sdv_tracker_get_cloud.argtypes = [_vp, C.c_int, C.c_int, C.POINTER(C.c_int), _vp, _vp, _vp, _vp]
    L.sdv_tracker_calc_res.argtypes = [_vp, C.c_int, C.c_uint64, C.c_int, _f64p, C.c_double, C.c_double, C.c_float, _f64p]
    L.sdv_tracker_calc_gs.argtypes = [_vp, C.c_int, C.c_int, _f64p, _f64p]
    L.sdv_reproject_grid.argtypes = [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.sdv_map_set.argtypes = [_vp, C.c_int, C.c_int, _u64p, _f64p, _f64p, C.c_int, _vp]
    L.sdv_tracker_set_ref_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _f32p, _i32p, _vp, _i32p]
    L.sdv_map_set_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _u64p, _f64p, _f64p, _i32p, _vp]
    L.sdv_reproject_map_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _f64p, _f64p, _i32p, _i32p, _i32p, _vp, C.c_int, _i32p, _i32p, _f64p]
    L.sdv_tracker_refine_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _f64p, _f64p, _vp, C.c_int, _i32p, _f32p, _i32p, _i32p]
    L.sdv_tracker_struct_pose_batch.argtypes = [_vp, C.c_int, _i32p, _vp, _i32p, _f64p, _f64p, _f32p, _i32p, _i32p]
    L.sdv_tracker_struct_pose_batch_slots.argtypes = [_vp, C.c_int, _vp, _i32p, _vp, _i32p, _f64p, _f64p, _f32p, _i32p, _i32p]
    L.sdv_tracker_track.argtypes = [_vp, C.c_int, C.c_uint64, _f64p, _f64p, C.c_int, _f64p, _f64p, _f64p, C.POINTER(C.c_int), C.POINTER(sdv_track_stats)]
    L.sdv_tracker_track_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _f64p, _f64p, C.c_int, _vp, _f64p, _f64p, _i32p, C.POINTER(sdv_track_stats)]
    L.sdv_tracker_track_batch_levels.argtypes = [_vp, C.c_int, _i32p, _u64p, _f64p, _f64p, _vp, _vp, _f64p, _f64p, _i32p, C.POINTER(sdv_track_stats)]
    L.sdv_last_kernel_ms.argtypes = [_vp]; L.sdv_last_kernel_ms.restype = C.c_float
    L.sdv_immature_init.argtypes = [_vp, C.c_uint64, C.c_int, _i32p, _vp]
    L.sdv_immature_trace_batch.argtypes = [_vp, C.c_int, _u64p, _i32p, _f32p, _f32p, _f32p, _vp, _vp]
    L.sdv_immature_optimize_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _u64p, _f32p, _f32p, C.c_int, _vp, _vp, C.c_int, _i32p, _f32p, _i32p]
    L.sdv_ba_last_kernel_ms.argtypes = [_vp]; L.sdv_ba_last_kernel_ms.restype = C.c_float
    L.sdv_selector_init.argtypes = [_vp, _vp, C.c_int]
    L.sdv_selector_potential.argtypes = [_vp, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.sdv_selector_get_map.argtypes = [_vp, C.c_int, _vp]
    L.sdv_selector_make_hists.argtypes = [_vp, C.c_uint64, _vp, _vp]
    L.sdv_selector_make_maps_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _vp, _vp, _f32p, _i32p, _f32p, _vp, _i32p]
    L.sdv_make_new_traces_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _vp, _f32p, _f32p, _i32p, C.c_int, _vp, _vp, _i32p, _i32p]
    L.sdv_lidar_init.argtypes = [_vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]
    L.sdv_lidar_handler_batch.argtypes = [_vp, C.c_int, _i32p, _vp, _f64p, _f64p, _f32p, _i32p, C.c_int, _vp, _i32p, _i32p, _i32p]
    L.sdv_activate_select_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _vp, _vp, _vp, _i32p, _i32p, _vp, _vp, _vp, _f32p, _vp, _vp]
    L.sdv_selector_set_slot_cams.argtypes = [_vp, C.c_int, _i32p, _i32p]
    L.sdv_selector_make_hists_cam.argtypes = [_vp, C.c_int, C.c_uint64, _vp, _vp]
    L.sdv_activate_select_batch_cams.argtypes = [_vp, C.c_int, _i32p, _i32p, _vp, _vp, _vp, _i32p, _i32p, _vp, _vp, _vp, _f32p, _vp, _vp, _vp]
    L.sdv_lidar_handler_batch_cams.argtypes = [_vp, C.c_int, _i32p, _vp, _f64p, _f64p, _f32p, _vp, _i32p, C.c_int, _vp, _i32p, _i32p, _i32p]
    L.sdv_immature_init_cam.argtypes = [_vp, C.c_int, C.c_uint64, C.c_int, _i32p, _vp]
    L.sdv_immature_trace_batch_cams.argtypes = [_vp, C.c_int, _u64p, _vp, _i32p, _f32p, _f32p, _f32p, _vp, _vp]
    L.sdv_immature_optimize_batch_cams.argtypes = [_vp, C.c_int, _i32p, _i32p, _u64p, _f32p, _f32p, _vp, C.c_int, _vp, _vp, C.c_int, _i32p, _f32p, _i32p]
    L.sdv_immature_store_set.argtypes = [_vp, C.c_uint64, C.c_int, _vp, _vp]
    L.sdv_immature_store_count.argtypes = [_vp, C.c_int, _u64p, _i32p]
    L.sdv_immature_store_get.argtypes = [_vp, C.c_uint64, C.c_int, _vp, _vp, C.POINTER(C.c_int32)]
    L.sdv_immature_store_drop.argtypes = [_vp, C.c_int, _u64p]
    L.sdv_immature_trace_store_batch.argtypes = [_vp, C.c_int, _u64p, _u64p, _vp, _f32p, _f32p, _f32p, _vp]
    L.sdv_activate_points_store_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _f32p, _f32p, _i32p, _i32p, _vp, _vp, _vp, _f32p, _f32p, _f32p, _vp, C.c_int, _i32p,
                                                  _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    L.sdv_make_new_traces_store_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _vp, _f32p, _f32p, _i32p, C.c_int, _i32p, _i32p]
    L.sdv_selector_lidar_box.argtypes = [_vp, C.c_int, _vp, _vp]
    L.sdv_lidar_handler_rows_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _vp, _f64p, _f64p, _f32p, C.c_int, _vp]
    L.sdv_lidar_rows_get.argtypes = [_vp, C.c_uint64, C.c_int, _vp, C.POINTER(C.c_int32), _vp, C.POINTER(C.c_int32)]
    L.sdv_lidar_rows_drop.argtypes = [_vp, C.c_int, _u64p]
    L.sdv_make_new_traces_rows_store_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _f32p, C.c_int, _i32p, _i32p]
    L.sdv_init_from_lidar_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _i32p, _vp, _i32p, _f32p, _i32p, _i32p, C.c_int, _i32p, _i32p, _vp, _vp, _vp]
    L.sdv_init_from_lidar_rows_batch.argtypes = [_vp, C.c_int, _i32p, _u64p, _f32p, _i32p, _i32p, C.c_int, _i32p, _i32p, _vp, _vp, _vp]
    return L


LIB = _load()


class SdvError(RuntimeError):
    pass


def track_job_bytes() -> int:
    """bytes copied H2D and D2H per trackNewestCoarse job descriptor"""
    return int(LIB.sdv_track_job_bytes())


def pyr_levels(w: int, h: int) -> int:
    return LIB.sdv_pyr_levels(w, h)


def default_settings() -> sdv_settings:
    s = sdv_settings(); LIB.sdv_default_settings(C.byref(s)); return s


class Context:
    def __init__(self, K, w: int, h: int, levels: int | None = None, device: int = 0, **settings):
        self.w, self.h = w, h
        self.cam_wh = {0: (w, h)}          # rectified size per camera (setCameraSize); camera 0 is the context size
        self.frame_cam = {}                # frame handle -> camera, for frames not on camera 0
        self.slot_cam = {}                 # tracker / map slot -> camera, for slots not on camera 0 (setCalibSlots)
        self.levels = levels if levels is not None else pyr_levels(w, h)     # storage depth: every frame is built to it
        self.cam_levels = {}               # pyramid depth per camera, for cameras not at the context's (setCameraLevels)
        s = default_settings()
        for k, v in settings.items():
            if not hasattr(s, k):
                raise TypeError(f"unknown setting {k}")
            setattr(s, k, v)
        self.settings = s
        cal = sdv_calib(*[float(k) for k in K])
        self.p = _vp()
        rc = LIB.sdv_create(C.byref(cal), w, h, self.levels, C.byref(s), device, C.byref(self.p))
        if rc != 0:
            msg = LIB.sdv_last_error(None).decode()      # no context exists after a failed create: the library keeps the message per thread
            self.p = None
            raise SdvError(f"sdv_create failed ({rc}): {msg}")

    def _ck(self, rc):
        if rc != 0:
            raise SdvError(f"sdv error {rc}: {LIB.sdv_last_error(self.p).decode()}")

    def close(self):
        if getattr(self, "p", None):
            LIB.sdv_destroy(self.p); self.p = None

    def __del__(self):
        self.close()

    def sync(self):
        self._ck(LIB.sdv_sync(self.p))

    def camSize(self, cam: int = 0):
        """(w, h) of camera `cam`'s frames"""
        return self.cam_wh.get(int(cam), (self.w, self.h))

    def setCameraSize(self, cam: int, w: int, h: int):
        """give camera `cam` (1..SDV_MAX_CAMERAS-1) the rectified size w x h <= the context size, at the context's pyramid depth (see sdv_b200.h)"""
        self._ck(LIB.sdv_set_camera_size(self.p, int(cam), int(w), int(h))); self.cam_wh[int(cam)] = (int(w), int(h))

    def setCameraStorage(self, cam: int, max_frames: int, max_kf_images: int = 0):
        """give camera `cam` (1..SDV_MAX_CAMERAS-1) its own pool of max_frames frames and max_kf_images keyframe level-0 images (0: the default) at its
        size; max_frames == 0 drops it (its frames come from the context pool again).  See sdv_b200.h"""
        self._ck(LIB.sdv_set_camera_storage(self.p, int(cam), int(max_frames), int(max_kf_images)))

    def cameraStorageBytes(self, cam: int = 0):
        """(frame_bytes, kf_image_bytes): device bytes of one frame and one keyframe level-0 image of camera `cam` as they are stored now"""
        fb, kb = C.c_uint64(), C.c_uint64()
        self._ck(LIB.sdv_camera_storage_bytes(self.p, int(cam), C.byref(fb), C.byref(kb)))
        return int(fb.value), int(kb.value)

    def camLevels(self, cam: int = 0) -> int:
        """pyramid depth (pyrLevelsUsed) of camera `cam`: what its tracker / map slots and jobs use"""
        return self.cam_levels.get(int(cam), self.levels)

    def setCameraLevels(self, cam: int, levels: int):
        """give camera `cam` (0..SDV_MAX_CAMERAS-1) the pyramid depth `levels` in 1..self.levels; the reference rule is pyr_levels(*camSize(cam)) (see sdv_b200.h)"""
        self._ck(LIB.sdv_set_camera_levels(self.p, int(cam), int(levels)))
        if int(levels) == self.levels:
            self.cam_levels.pop(int(cam), None)
        else:
            self.cam_levels[int(cam)] = int(levels)

    def _check_level(self, lvl: int, cam: int, what: str):
        if not 0 <= lvl < self.camLevels(cam):
            raise SdvError(f"sdv error -1: {what}: level {lvl}, but camera {cam} has {self.camLevels(cam)} levels")

    # FrameHessian::makeImages
    def makeImages(self, frame_id: int, color, exposure: float = 1.0, cam: int = 0):
        color = np.ascontiguousarray(color, np.float32)
        w, h = self.camSize(cam)
        assert color.shape == (h, w), f"camera {cam} takes {w}x{h} images"
        if cam == 0:
            self._ck(LIB.sdv_frame_upload(self.p, frame_id, color.ctypes.data, exposure)); self.frame_cam.pop(frame_id, None)
        else:
            self.makeImagesBatch([frame_id], [color.ctypes.data], [exposure], cams=[cam]); self.sync()

    def setCalib(self, K):
        """CoarseTracker::makeK / the CalibHessian the Reprojector reads, after the bundle adjustment moved the intrinsics"""
        k = sdv_calib(*[float(x) for x in K]); self._ck(LIB.sdv_set_calib(self.p, C.byref(k))); self.K = tuple(float(x) for x in K)

    def setCalibSlots(self, slots, Ks, cams=None):
        """CoarseTracker::makeK per tracker instance: slot slots[i] (its tracker and the map slot of the same index) uses Ks[i] = (fx, fy, cx, cy) from now on,
        whatever setCalib sets later, and is bound to camera cams[i] (None: camera 0): its frames must have that camera's size.
        All-or-nothing: a bad slot, K or camera raises SdvError and changes no slot."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1); Kf = np.asarray(Ks, np.float64).reshape(-1, 4)
        if len(Kf) != len(sl):
            raise ValueError(f"{len(sl)} slots but {len(Kf)} calibrations")
        cm = self._cams(cams, len(sl))
        arr = (sdv_calib * max(len(sl), 1))(*[sdv_calib(*map(float, k)) for k in Kf])
        self._ck(LIB.sdv_set_calib_slots_cams(self.p, len(sl), sl, C.addressof(arr), None if cm is None else cm.ctypes.data))
        self._bind(sl, cm)

    def _bind(self, sl, cm):
        for s, c in zip(sl.tolist(), [0] * len(sl) if cm is None else cm.tolist()):
            if c:
                self.slot_cam[s] = c
            else:
                self.slot_cam.pop(s, None)

    @staticmethod
    def _cams(cams, n):
        if cams is None:
            return None
        cm = np.ascontiguousarray(cams, np.int32).reshape(-1)
        if len(cm) != n:
            raise ValueError(f"{n} entries but {len(cm)} camera indices")
        return cm

    def clearCalibSlots(self, slots):
        """the slots follow the context calibration (setCalib) again"""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        self._ck(LIB.sdv_set_calib_slots(self.p, len(sl), sl, None)); self._bind(sl, None)

    # Undistort (util/Undistort.cpp) handed over as data; `und` = sdv_loam_b200.undistort.Undistort or anything with wOrg,hOrg,remapX,remapY[,G,vignetteMapInv]
    # cam: which of the context's SDV_MAX_CAMERAS cameras these tables set or replace (the raw size is per camera, the rectified size is the camera's: setCameraSize)
    def setUndistort(self, und, factor: float = 1.0, cam: int = 0):
        rx = np.ascontiguousarray(und.remapX, np.float32).reshape(-1); ry = np.ascontiguousarray(und.remapY, np.float32).reshape(-1)
        w, h = self.camSize(cam)
        assert rx.size == w * h == ry.size, f"remap tables must have camera {cam}'s rectified size {w}x{h}"
        G = getattr(und, "G", None); V = getattr(und, "vignetteMapInv", None)
        G = None if G is None else np.ascontiguousarray(G, np.float32); V = None if V is None else np.ascontiguousarray(V, np.float32)
        assert G is None or G.size == 256
        assert V is None or V.size == und.wOrg * und.hOrg
        self._ck(LIB.sdv_set_undistort_cam(self.p, int(cam), int(und.wOrg), int(und.hOrg), rx, ry, float(factor), None if G is None else G.ctypes.data, None if V is None else V.ctypes.data))
        self.wh_org = getattr(self, "wh_org", {}); self.wh_org[int(cam)] = (int(und.wOrg), int(und.hOrg))

    def setGammaFunction(self, BInv, cam: int = 0):
        """FullSystem::setGammaFunction for camera `cam`: BInv = PhotometricUndistorter.getG() (at least 256 values, the first 256 are read), or None for the
        identity.  The frames of this camera then carry makeImages' gamma-weighted absSquaredGrad (sdv_set_gamma_cam).  Call it before the camera's first frame."""
        if BInv is None:
            self._ck(LIB.sdv_set_gamma_cam(self.p, int(cam), None)); return
        b = np.ascontiguousarray(np.asarray(BInv, np.float32).reshape(-1)[:256])
        if b.size != 256:
            raise ValueError(f"setGammaFunction reads 256 values, got {b.size}")
        self._ck(LIB.sdv_set_gamma_cam(self.p, int(cam), b.ctypes.data))

    def setCameraPhotometric(self, und, factor: float = 1.0, cam: int = 0):
        """what src/main.cpp does for a camera: its Undistort (with the PhotometricUndistorter attached by Undistort.set_photometric, if any) for the raw
        ingest, then FullSystem::setGammaFunction(getPhotometricGamma()), which is None (identity) without a valid photometric calibration"""
        self.setUndistort(und, factor, cam)
        pu = getattr(und, "photometricUndist", None)
        self.setGammaFunction(None if pu is None else pu.getG(), cam)

    def makeImagesRaw(self, frame_id: int, raw, exposure: float = 1.0, cam: int = 0):
        """Undistort::undistort<unsigned char> + FrameHessian::makeImages of one native-size mono8 image of camera `cam`"""
        raw = np.ascontiguousarray(raw, np.uint8); cam = int(cam)
        if cam in getattr(self, "wh_org", {}):
            assert raw.shape == (self.wh_org[cam][1], self.wh_org[cam][0]), f"camera {cam} takes {self.wh_org[cam][0]}x{self.wh_org[cam][1]} images"
        self.makeImagesBatch([frame_id], [raw.ctypes.data], [exposure], raw=True, cams=[cam]); self.sync()

    def makeImagesBatch(self, frame_ids, ptrs, exposures=None, u8=False, device=False, adopt=False, raw=False, cams=None):
        """Batched makeImages.  ptrs: integer addresses of (h,w) buffers — host (pinned for full-rate, asynchronous H2D)
        or device (device=True); float32, or mono8 when u8=True; raw=True: native-size mono8 through setUndistort's tables.
        Image k is camera cams[k] (None: every image is camera 0) and has that camera's size (raw: its raw size).
        A uint64 numpy array of addresses avoids per-call list work.  Asynchronous: see sdv_b200.h."""
        n = len(frame_ids)
        ids = np.ascontiguousarray(frame_ids, np.uint64)
        if isinstance(ptrs, np.ndarray):
            parr = np.ascontiguousarray(ptrs, np.uint64); arr = parr.ctypes.data_as(C.POINTER(_vp))
        else:
            arr = (_vp * n)(*ptrs)
        ex = self._ones(n) if exposures is None else np.ascontiguousarray(exposures, np.float32)
        cm = self._cams(cams, n)
        if cm is not None:
            if raw:
                self._ck(LIB.sdv_frame_upload_batch_raw_u8_cams(self.p, n, ids, arr, cm.ctypes.data, ex))
            elif device:
                self._ck(LIB.sdv_frame_build_batch_dev_cams(self.p, n, ids, arr, cm.ctypes.data, 1 if u8 else (2 if adopt else 0), ex))
            else:
                self._ck(LIB.sdv_frame_upload_batch_cams(self.p, n, ids, arr, cm.ctypes.data, 1 if u8 else 0, ex))
            for i, k in zip(ids.tolist(), cm.tolist()):
                if k:
                    self.frame_cam[i] = k
                else:
                    self.frame_cam.pop(i, None)
            return
        if self.frame_cam:                 # these handles are camera-0 frames now
            for i in ids.tolist():
                self.frame_cam.pop(i, None)
        if raw:
            self._ck(LIB.sdv_frame_upload_batch_raw_u8(self.p, n, ids, arr, ex))
        elif device:
            self._ck(LIB.sdv_frame_build_batch_dev(self.p, n, ids, arr, 1 if u8 else (2 if adopt else 0), ex))
        elif u8:
            self._ck(LIB.sdv_frame_upload_batch_u8(self.p, n, ids, arr, ex))
        else:
            self._ck(LIB.sdv_frame_upload_batch(self.p, n, ids, arr, ex))

    def _ones(self, n):
        o = getattr(self, "_ones_cache", None)
        if o is None or len(o) != n:
            o = self._ones_cache = np.ones(n, np.float32)
        return o

    def launch_count(self) -> int:
        return int(LIB.sdv_launch_count(self.p))

    def ba_host_wait_count(self) -> int:
        """host waits on the back-end stream so far (sdv_ba_host_wait_count)"""
        LIB.sdv_ba_host_wait_count.argtypes = [_vp]; LIB.sdv_ba_host_wait_count.restype = C.c_longlong
        return int(LIB.sdv_ba_host_wait_count(self.p))

    def releaseFrame(self, frame_id: int):
        self._ck(LIB.sdv_frame_release(self.p, frame_id)); self.frame_cam.pop(frame_id, None)

    def frameLevel(self, frame_id: int, lvl: int):
        """level lvl (below its camera's depth) of a resident frame at the frame's own (its camera's) size"""
        cam = self.frame_cam.get(frame_id, 0); self._check_level(lvl, cam, "frameLevel")
        w, h = self.camSize(cam); w, h = w >> lvl, h >> lvl
        dI = np.zeros((h, w, 3), np.float32); ab = np.zeros((h, w), np.float32)
        self._ck(LIB.sdv_frame_download(self.p, frame_id, lvl, dI.ctypes.data, ab.ctypes.data))
        return dI, ab

    def last_kernel_ms(self) -> float:
        return float(LIB.sdv_last_kernel_ms(self.p))

    def trackBatch(self, slots, frame_ids, T, ab, coarsest=None, minRes=None):
        """n independent trackNewestCoarse calls in one launch.  T (n,7), ab (n,2) are updated in place.
        coarsest: None starts each job at its slot camera's depth - 1 (pyrLevelsUsed-1); an int is that level for every job; a sequence one level per job.
        slots / frame_ids may be pre-built contiguous int32 / uint64 arrays (no per-call Python work beyond the C call)."""
        n = len(slots)
        slots = np.ascontiguousarray(slots, np.int32); ids = np.ascontiguousarray(frame_ids, np.uint64)
        assert T.dtype == np.float64 and T.shape == (n, 7) and T.flags.c_contiguous
        assert ab.dtype == np.float64 and ab.shape == (n, 2) and ab.flags.c_contiguous
        lastRes = np.empty((n, 5)); flow = np.empty((n, 3)); good = np.empty(n, np.int32)
        stats = np.empty(n, TRACK_STATS_DTYPE)
        mr = None if minRes is None else np.ascontiguousarray(minRes, np.float64).ctypes.data
        sp = stats.ctypes.data_as(C.POINTER(sdv_track_stats))
        if isinstance(coarsest, (int, np.integer)):
            self._ck(LIB.sdv_tracker_track_batch(self.p, n, slots, ids, T, ab, int(coarsest), mr, lastRes, flow, good, sp))
        else:
            co = None if coarsest is None else np.ascontiguousarray(coarsest, np.int32).reshape(-1)
            if co is not None and len(co) != n:
                raise ValueError(f"{n} jobs but {len(co)} coarsest levels")
            self._ck(LIB.sdv_tracker_track_batch_levels(self.p, n, slots, ids, T, ab, None if co is None else co.ctypes.data, mr, lastRes, flow, good, sp))
        return dict(good=good.astype(bool), lastResiduals=lastRes, flow=flow, evals=stats["point_evals"], iterations=stats["iterations"], accepts=stats["accepts"])

    def setCoarseTrackingRefBatch(self, slots, frame_ids, pts_list, round_half_list, ref_ab=None):
        """CoarseTracker::setCoarseTrackingRef for n tracker slots in one call (sdv_tracker_set_ref_batch): slot slots[j] gets the reference frame frame_ids[j]
        and the splat rows pts_list[j] ({u, v, idepth, HdiF}) with round_half_list[j]; ref_ab (n, 2) or None = (0, 0).  Returns the (n, levels) cloud sizes.
        Over max_ref_points raises SdvError after installing every job that fits (see sdv_b200.h)."""
        n = len(slots); sl = np.ascontiguousarray(slots, np.int32).reshape(-1); fr = np.ascontiguousarray(frame_ids, np.uint64).reshape(-1)
        P = [np.ascontiguousarray(p, np.float32).reshape(-1, 4) for p in pts_list]; R = [np.ascontiguousarray(r, np.int32).reshape(-1) for r in round_half_list]
        if not (len(sl) == len(fr) == len(P) == len(R) == n) or any(len(p) != len(r) for p, r in zip(P, R)):
            raise ValueError("setCoarseTrackingRefBatch: one frame, one row array and one round_half array per slot, of equal lengths")
        pb = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(p) for p in P], dtype=np.int64)]), np.int32)
        p4 = np.ascontiguousarray(np.concatenate(P) if pb[-1] else np.zeros((1, 4)), np.float32); rh = np.ascontiguousarray(np.concatenate(R) if pb[-1] else np.zeros(1), np.int32)
        ab = None if ref_ab is None else np.ascontiguousarray(ref_ab, np.float64).reshape(n, 2)
        out = np.zeros((max(n, 1), PYR_LEVELS), np.int32)
        self._ck(LIB.sdv_tracker_set_ref_batch(self.p, n, sl, fr, pb, p4, rh, None if ab is None else ab.ctypes.data, out))
        return out[:n, :self.levels]


class CoarseTracker:
    """Mirror of sdv_loam::CoarseTracker (FullSystem/CoarseTracker.h:16-133) bound to one tracker slot of a Context."""

    def __init__(self, ctx: Context, slot: int = 0):
        self.ctx, self.slot = ctx, slot

    @property
    def levels(self) -> int:
        """pyrLevelsUsed of this instance: its slot camera's depth"""
        return self.ctx.camLevels(self.ctx.slot_cam.get(self.slot, 0))

    def _check_level(self, lvl: int, what: str):
        self.ctx._check_level(lvl, self.ctx.slot_cam.get(self.slot, 0), what)

    def makeK(self, K):
        """CoarseTracker::makeK (CoarseTracker.cpp:77-106): this instance tracks (and refines its slot's map) with K = (fx, fy, cx, cy) from now on,
        on the camera its slot is bound to"""
        self.ctx.setCalibSlots([self.slot], [K], cams=[self.ctx.slot_cam.get(self.slot, 0)])

    def setCoarseTrackingRef(self, ref_frame_id: int, pts, round_half, ref_a: float = 0.0, ref_b: float = 0.0):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4); rh = np.ascontiguousarray(round_half, np.int32)
        self.ctx._ck(LIB.sdv_tracker_set_ref(self.ctx.p, self.slot, ref_frame_id, len(pts), pts, rh, 0.0, ref_a, ref_b))

    def setCloud(self, ref_frame_id: int, lvl: int, u, v, idepth, color, ref_a: float = 0.0, ref_b: float = 0.0):
        self._check_level(lvl, "setCloud"); a = [np.ascontiguousarray(x, np.float32) for x in (u, v, idepth, color)]
        self.ctx._ck(LIB.sdv_tracker_set_cloud(self.ctx.p, self.slot, ref_frame_id, lvl, len(a[0]), *a, ref_a, ref_b))

    def cloud(self, lvl: int):
        self._check_level(lvl, "cloud"); n = C.c_int(0)
        self.ctx._ck(LIB.sdv_tracker_get_cloud(self.ctx.p, self.slot, lvl, C.byref(n), None, None, None, None))
        a = [np.zeros(max(n.value, 1), np.float32) for _ in range(4)]
        self.ctx._ck(LIB.sdv_tracker_get_cloud(self.ctx.p, self.slot, lvl, C.byref(n), *[x.ctypes.data for x in a]))
        return [x[:n.value] for x in a]

    def calcRes(self, new_frame_id: int, lvl: int, T7, a: float, b: float, cutoffTH: float):
        self._check_level(lvl, "calcRes"); rs = np.zeros(6)
        self.ctx._ck(LIB.sdv_tracker_calc_res(self.ctx.p, self.slot, new_frame_id, lvl, np.ascontiguousarray(T7, np.float64), a, b, cutoffTH, rs))
        return rs

    def calcGSSSE(self, lvl: int):
        H = np.zeros(64); b = np.zeros(8)
        self.ctx._ck(LIB.sdv_tracker_calc_gs(self.ctx.p, self.slot, lvl, H, b))
        return H.reshape(8, 8), b

    def trackNewestCoarse(self, new_frame_id: int, T7, ab, coarsest=None, minRes=None):
        T = np.array(T7, np.float64).reshape(1, 7); abv = np.array(ab, np.float64).reshape(1, 2)
        mr = None if minRes is None else np.asarray(minRes, np.float64).reshape(1, 5)
        r = self.ctx.trackBatch([self.slot], [new_frame_id], T, abv, coarsest, mr)
        return dict(good=bool(r["good"][0]), T=T[0], ab=abv[0], lastResiduals=r["lastResiduals"][0], flow=r["flow"][0],
                    evals=r["evals"][0], iterations=r["iterations"][0], accepts=r["accepts"][0])

    def structPoseEstimation(self, curToWorld7, overlap_pts, host_T7):
        """CoarseTracker::structPoseEstimation (CoarseTracker.cpp:949-1007).  overlap_pts: OVERLAP_PT_DTYPE array, host_T7: (nH,7) camToWorld of
        the host keyframes the points index.  Returns dict(T=refined curToWorld, res, iterations, accepts)."""
        r = structPoseEstimationBatch(self.ctx, np.array(curToWorld7, np.float64).reshape(1, 7), [overlap_pts], [host_T7], slots=[self.slot])
        return dict(T=r["T"][0], res=float(r["res"][0]), iterations=int(r["iterations"][0]), accepts=int(r["accepts"][0]))


class sdv_track_new_coarse_io(C.Structure):
    _fields_ = [("slot", C.c_int32), ("poses_valid", C.c_int32), ("frame", C.c_uint64), ("sprelast_c2w", C.c_double * 7), ("slast_c2w", C.c_double * 7), ("lastF_c2w", C.c_double * 7),
                ("aff_last", C.c_double * 2), ("lastCoarseRMSE", C.c_double * 5), ("camToWorld", C.c_double * 7), ("camToTrackingRef", C.c_double * 7), ("aff_g2l", C.c_double * 2),
                ("flow", C.c_double * 3), ("refine_res", C.c_float), ("have_one_good", C.c_int32), ("tries", C.c_int32), ("n_matches", C.c_int32), ("refine_iterations", C.c_int32),
                ("refine_accepts", C.c_int32)]


TRACK_NEW_COARSE_DTYPE = np.dtype([("slot", np.int32), ("poses_valid", np.int32), ("frame", np.uint64), ("sprelast_c2w", np.float64, 7), ("slast_c2w", np.float64, 7),
                                   ("lastF_c2w", np.float64, 7), ("aff_last", np.float64, 2), ("lastCoarseRMSE", np.float64, 5), ("camToWorld", np.float64, 7),
                                   ("camToTrackingRef", np.float64, 7), ("aff_g2l", np.float64, 2), ("flow", np.float64, 3), ("refine_res", np.float32),
                                   ("have_one_good", np.int32), ("tries", np.int32), ("n_matches", np.int32), ("refine_iterations", np.int32), ("refine_accepts", np.int32)], align=True)
assert TRACK_NEW_COARSE_DTYPE.itemsize == C.sizeof(sdv_track_new_coarse_io)


def trackNewCoarseBatchArray(ctx, io, cell_order=None, max_matches=400):
    """Same as trackNewCoarseBatch on a numpy structured array (TRACK_NEW_COARSE_DTYPE), updated in place — no per-job Python work."""
    LIB.sdv_track_new_coarse_batch.argtypes = [_vp, C.c_int, _vp, _vp, C.c_int]
    assert io.dtype == TRACK_NEW_COARSE_DTYPE and io.flags.c_contiguous
    co = None if cell_order is None else np.ascontiguousarray(cell_order, np.int32)
    ctx._ck(LIB.sdv_track_new_coarse_batch(ctx.p, len(io), io.ctypes.data, None if co is None else co.ctypes.data, max_matches))
    return io


def trackNewCoarseBatch(ctx, jobs, cell_order=None, max_matches=400):
    """FullSystem::trackNewCoarse (FullSystem.cpp:283-500) for n sequences.  jobs: dicts with slot, frame, sprelast_c2w, slast_c2w, lastF_c2w, aff_last,
    poses_valid, lastCoarseRMSE.  Returns one dict per job with the fields of sdv_track_new_coarse_io."""
    LIB.sdv_track_new_coarse_batch.argtypes = [_vp, C.c_int, _vp, _vp, C.c_int]
    n = len(jobs); io = (sdv_track_new_coarse_io * n)()
    for k, j in enumerate(jobs):
        io[k].slot = j["slot"]; io[k].poses_valid = int(j.get("poses_valid", 1)); io[k].frame = j["frame"]
        for name in ("sprelast_c2w", "slast_c2w", "lastF_c2w", "aff_last", "lastCoarseRMSE"):
            v = np.asarray(j[name], np.float64); getattr(io[k], name)[:] = v.tolist()
    co = None if cell_order is None else np.ascontiguousarray(cell_order, np.int32)
    ctx._ck(LIB.sdv_track_new_coarse_batch(ctx.p, n, C.addressof(io), None if co is None else co.ctypes.data, max_matches))
    out = []
    for k in range(n):
        o = io[k]
        out.append(dict(camToWorld=np.array(o.camToWorld[:]), camToTrackingRef=np.array(o.camToTrackingRef[:]), aff_g2l=np.array(o.aff_g2l[:]), flow=np.array(o.flow[:]),
                        lastCoarseRMSE=np.array(o.lastCoarseRMSE[:]), have_one_good=bool(o.have_one_good), tries=int(o.tries), n_matches=int(o.n_matches),
                        refine_iterations=int(o.refine_iterations), refine_accepts=int(o.refine_accepts), refine_res=float(o.refine_res)))
    return out


class Reprojector:
    """Mirror of sdv_loam::Reprojector (FullSystem/Reprojector.h:17-111) over device-resident maps: one map slot per sequence."""

    def __init__(self, ctx: Context):
        self.ctx = ctx; a = C.c_int(0); b = C.c_int(0); ctx._ck(LIB.sdv_reproject_grid(ctx.p, C.byref(a), C.byref(b)))
        self.grid_n_cols, self.grid_n_rows = a.value, b.value; self.n_cells = a.value * b.value

    def setMap(self, slot: int, host_frame_ids, host_T7, host_ab, pts):
        pts = np.ascontiguousarray(pts, MAP_PT_DTYPE); hT = np.ascontiguousarray(host_T7, np.float64).reshape(-1, 7)
        hab = np.zeros((len(hT), 2)) if host_ab is None else np.ascontiguousarray(host_ab, np.float64).reshape(-1, 2)
        self.ctx._ck(LIB.sdv_map_set(self.ctx.p, slot, len(hT), np.ascontiguousarray(host_frame_ids, np.uint64), hT, hab, len(pts), pts.ctypes.data if len(pts) else None))

    def setMapBatch(self, slots, host_frame_ids_list, host_T7_list, host_ab_list, pts_list):
        """setMap for n slots in one call (sdv_map_set_batch): job j has the keyframes host_frame_ids_list[j] with host_T7_list[j] and host_ab_list[j] (None: all
        (0, 0); host_ab_list itself may be None) and the points pts_list[j] (MAP_PT_DTYPE, host indexing the job's keyframes).  All-or-nothing."""
        n = len(slots); sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        ids = [np.ascontiguousarray(f, np.uint64).reshape(-1) for f in host_frame_ids_list]; T = [np.ascontiguousarray(t, np.float64).reshape(-1, 7) for t in host_T7_list]
        abl = [None] * n if host_ab_list is None else host_ab_list
        AB = [np.zeros((len(t), 2)) if a is None else np.ascontiguousarray(a, np.float64).reshape(-1, 2) for a, t in zip(abl, T)]
        P = [np.ascontiguousarray(p, MAP_PT_DTYPE).reshape(-1) for p in pts_list]
        if not (len(sl) == len(ids) == len(T) == len(AB) == len(P) == n):
            raise ValueError("setMapBatch: one keyframe list, pose list, ab list and point array per slot")
        cum = lambda a: np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(x) for x in a], dtype=np.int64)]), np.int32)
        hb, pb = cum(ids), cum(P)
        cat = lambda a, empty: np.ascontiguousarray(np.concatenate(a) if sum(len(x) for x in a) else empty)
        pts = cat(P, np.zeros(1, MAP_PT_DTYPE))
        self.ctx._ck(LIB.sdv_map_set_batch(self.ctx.p, n, sl, hb, cat(ids, np.zeros(1, np.uint64)), cat(T, np.zeros((1, 7))), cat(AB, np.zeros((1, 2))), pb, pts.ctypes.data))

    def reprojectMapBatch(self, slots, cur_frame_ids, cur_T7, cur_ab=None, cur_kf_index=None, only_host=None, backup=None, cell_order=None, max_matches=400):
        n = len(slots); i32 = lambda a, d: np.full(n, d, np.int32) if a is None else np.ascontiguousarray(a, np.int32)
        T = np.ascontiguousarray(cur_T7, np.float64).reshape(n, 7); ab = np.zeros((n, 2)) if cur_ab is None else np.ascontiguousarray(cur_ab, np.float64).reshape(n, 2)
        n_out = np.zeros(n, np.int32); out_pt = np.zeros((n, self.n_cells), np.int32); out_px = np.zeros((n, self.n_cells, 2))
        co = None if cell_order is None else np.ascontiguousarray(cell_order, np.int32)
        self.ctx._ck(LIB.sdv_reproject_map_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(cur_frame_ids, np.uint64), T, ab,
                                                 i32(cur_kf_index, -1), i32(only_host, -1), i32(backup, 0), None if co is None else co.ctypes.data, max_matches, n_out, out_pt, out_px))
        return [(out_pt[k, :n_out[k]].copy(), out_px[k, :n_out[k]].copy()) for k in range(n)]

    def refineBatch(self, slots, cur_frame_ids, curToWorld7, cur_ab=None, cell_order=None, max_matches=400):
        """Tail of FullSystem::trackNewCoarse (FullSystem.cpp:482-488) for n frames: reprojectMap -> structPoseEstimation, device resident."""
        n = len(slots); T = np.ascontiguousarray(curToWorld7, np.float64).reshape(n, 7).copy()
        ab = np.zeros((n, 2)) if cur_ab is None else np.ascontiguousarray(cur_ab, np.float64).reshape(n, 2)
        co = None if cell_order is None else np.ascontiguousarray(cell_order, np.int32)
        nm = np.zeros(n, np.int32); res = np.zeros(n, np.float32); its = np.zeros(n, np.int32); acc = np.zeros(n, np.int32)
        self.ctx._ck(LIB.sdv_tracker_refine_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(cur_frame_ids, np.uint64), T, ab,
                                                  None if co is None else co.ctypes.data, max_matches, nm, res, its, acc))
        return dict(T=T, n_matches=nm, res=res, iterations=its, accepts=acc, ms=self.ctx.last_kernel_ms())

    def reprojectMap(self, slot, cur_frame_id, cur_T7, cur_ab=None, **kw):
        kw = {k: (None if v is None else ([v] if k != "cell_order" and k != "max_matches" else v)) for k, v in kw.items()}
        return self.reprojectMapBatch([slot], [cur_frame_id], np.asarray(cur_T7, np.float64).reshape(1, 7), None if cur_ab is None else np.asarray(cur_ab, np.float64).reshape(1, 2), **kw)[0]


def structPoseEstimationBatch(ctx, curToWorld7, overlap_pts_list, host_T7_list, slots=None):
    """n independent structPoseEstimation calls in one launch (one CTA each): curToWorld7 (n,7) is refined in place.
    slots: the tracker slot of each job, whose K it uses (None: the context calibration)."""
    n = len(overlap_pts_list)
    T = np.ascontiguousarray(curToWorld7, np.float64).reshape(n, 7)
    pb = np.zeros(n + 1, np.int32); hb = np.zeros(n + 1, np.int32)
    pb[1:] = np.cumsum([len(p) for p in overlap_pts_list]); hb[1:] = np.cumsum([len(np.asarray(h).reshape(-1, 7)) for h in host_T7_list])
    pts = np.concatenate([np.ascontiguousarray(p, OVERLAP_PT_DTYPE) for p in overlap_pts_list]) if pb[-1] else np.zeros(1, OVERLAP_PT_DTYPE)
    hT = np.ascontiguousarray(np.concatenate([np.asarray(h, np.float64).reshape(-1, 7) for h in host_T7_list]))
    res = np.zeros(n, np.float32); its = np.zeros(n, np.int32); acc = np.zeros(n, np.int32)
    sl = None if slots is None else np.ascontiguousarray(slots, np.int32)
    assert sl is None or sl.shape == (n,)
    ctx._ck(LIB.sdv_tracker_struct_pose_batch_slots(ctx.p, n, None if sl is None else sl.ctypes.data, pb, pts.ctypes.data, hb, hT, T, res, its, acc))
    return dict(T=T, res=res, iterations=its, accepts=acc)


# ------------------------------------------------------------------------------------------------ back-end
def _ba_protos():
    L = LIB
    if getattr(L, "_ba_done", False):
        return
    L.sdv_ba_set_window.argtypes = [_vp, C.c_int, _u64p, _f64p, _f64p, _f64p, _f32p, _i32p, _f32p, _f64p, _f64p, _f64p]
    L.sdv_ba_set_points.argtypes = [_vp, C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p, _i32p, _i32p, _i32p, _i32p, C.c_int, _i32p, _i32p, _i32p, _i32p, _f32p, _i32p]
    L.sdv_ba_reset_oob.argtypes = [_vp]; L.sdv_ba_apply_res.argtypes = [_vp]; L.sdv_ba_backup.argtypes = [_vp]
    L.sdv_ba_linearize.argtypes = [_vp, C.c_int, C.POINTER(C.c_double)]
    L.sdv_ba_energy.argtypes = [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.sdv_ba_solve.argtypes = [_vp, C.c_int, C.c_double, _f64p]
    L.sdv_ba_step.argtypes = [_vp, C.c_float, C.c_int, C.POINTER(C.c_int)]
    L.sdv_ba_optimize.argtypes = [_vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.sdv_ba_select.argtypes = [_vp, C.c_int]
    L.sdv_ba_optimize_batch.argtypes = [_vp, C.c_int, _i32p, C.c_int, _f32p, _i32p, _i32p]
    L.sdv_ba_get_frames.argtypes = [_vp, _f64p, _f64p, _f64p, _f32p, _f64p, _f64p, _f64p]
    L.sdv_ba_get_points.argtypes = [_vp, _f32p, _f32p, _f32p, _f32p, _f32p, _i32p, _f32p]
    L.sdv_ba_get_residuals.argtypes = [_vp, _i32p, _i32p, _f32p, _i32p, _f32p, _f32p, _f32p, _f32p, _i32p]
    L.sdv_ba_get_system.argtypes = [_vp, _f64p, _f64p, _f64p, _f64p, _f64p, _f64p]
    L.sdv_ba_get_precalc.argtypes = [_vp, C.c_int, C.c_int, _f32p, _f64p, _f64p, _f32p]
    L.sdv_ba_flag_points.argtypes = [_vp, _i32p, _i32p]
    L.sdv_ba_marginalize_points.argtypes = [_vp, _vp]
    L.sdv_ba_marginalize_frame.argtypes = [_vp, C.c_int]
    L.sdv_ba_get_prior.argtypes = [_vp, C.POINTER(C.c_int), _vp, _vp]
    L.sdv_ba_get_linearized.argtypes = [_vp, _f32p, _i32p]
    L.sdv_ba_set_window_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _u64p, _f64p, _f64p, _f64p, _f32p, _i32p, _f32p, _f64p, _vp, _vp, _vp]
    L.sdv_ba_set_points_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _i32p] + [_f32p] * 5 + [_i32p] * 4 + [_i32p] * 4 + [_f32p, _i32p]
    L.sdv_ba_flag_points_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _vp]
    L.sdv_ba_marginalize_points_batch.argtypes = [_vp, C.c_int, _i32p, _vp]
    L.sdv_ba_marginalize_frames_batch.argtypes = [_vp, C.c_int, _i32p, _i32p, _i32p, _vp, _vp]
    L._ba_done = True


def _cat(arrs, dtype):
    a = [np.ascontiguousarray(x, dtype).reshape(-1) for x in arrs]
    return np.concatenate(a) if a else np.zeros(0, dtype)


def pack_ba_windows(wins, frame_ids_list):
    """The window dicts (synth.make_ba_window's layout) of one sdv_ba_set_window_batch / sdv_ba_set_points_batch call, concatenated in list order:
    f_begin / p_begin / r_begin (n + 1 each), the per-frame, per-point and per-residual arrays, res_begin blocks of nP_i + 1 entries each, calib_value_scaled
    and calib_value_zero (4 per window; the latter None unless some window has "K_zero", and for the others value_zero = value = value_scaled * (1.0f/50.0f) as the library forms it) and HM / bM (None unless some
    window has a prior; zero for the others, dim = 4 + 6 nF_i)."""
    n = len(wins); assert len(frame_ids_list) == n
    nF = np.array([int(w["nF"]) for w in wins], np.int64); nP = np.array([len(w["uv"]) for w in wins], np.int64); nR = np.array([len(w["r_point"]) for w in wins], np.int64)
    beg = lambda v: np.concatenate([[0], np.cumsum(v)]).astype(np.int32)
    for w, f in zip(wins, frame_ids_list):
        assert len(f) == int(w["nF"])
    o = dict(n=n, f_begin=beg(nF), p_begin=beg(nP), r_begin=beg(nR), frame_ids=_cat(frame_ids_list, np.uint64))
    for k, t in (("T_eval", np.float64), ("state", np.float64), ("state_zero", np.float64), ("ab_exposure", np.float32), ("frameID", np.int32), ("frameEnergyTH", np.float32),
                 ("uv", np.float32), ("idepth", np.float32), ("idepth_zero", np.float32), ("color", np.float32), ("weights", np.float32), ("host", np.int32),
                 ("hasDepthPrior", np.int32), ("isFromSensor", np.int32), ("res_begin", np.int32), ("r_point", np.int32), ("r_host", np.int32), ("r_target", np.int32),
                 ("r_hasMatcher", np.int32), ("r_matcher", np.float32), ("r_isNew", np.int32)):
        o[k] = _cat([w[k] for w in wins], t)
    o["K"] = _cat([w["K"] for w in wins], np.float64)
    zero = any("K_zero" in w for w in wins)
    o["K_zero"] = _cat([w["K_zero"] if "K_zero" in w else np.asarray(w["K"], np.float64) * np.float64(np.float32(1) / np.float32(50)) for w in wins], np.float64) if zero else None
    prior = any(w.get("HM") is not None for w in wins)
    dims = [4 + 6 * int(w["nF"]) for w in wins]
    o["HM"] = _cat([w["HM"] if w.get("HM") is not None else np.zeros((d, d)) for w, d in zip(wins, dims)], np.float64) if prior else None
    o["bM"] = _cat([w["bM"] if w.get("bM") is not None else np.zeros(d) for w, d in zip(wins, dims)], np.float64) if prior else None
    return o


class EnergyFunctional:
    """Mirror of the reference back-end surface (OptimizationBackend/EnergyFunctional.h:51-72 + FullSystem::optimize/linearizeAll)
    over a flattened window dict (see sdv_b200.h; synth.make_ba_window builds one).  frame_ids[i] = device frame handle of KF i."""

    def __init__(self, ctx: Context, win: dict, frame_ids, window: int = 0):
        _ba_protos(); self.ctx = ctx; self.win = win; self.window = window
        ctx._ck(LIB.sdv_ba_select(ctx.p, window))
        self.nF = win["nF"]; self.nP = len(win["uv"]); self.nR = len(win["r_point"]); self.n = 4 + 6 * self.nF
        c = lambda k, t: np.ascontiguousarray(win[k], t)
        ctx._ck(LIB.sdv_ba_set_window(ctx.p, self.nF, np.ascontiguousarray(frame_ids, np.uint64), c("T_eval", np.float64), c("state", np.float64),
                                      c("state_zero", np.float64), c("ab_exposure", np.float32), c("frameID", np.int32), c("frameEnergyTH", np.float32),
                                      c("K", np.float64), c("HM", np.float64), c("bM", np.float64)))
        if "K_zero" in win:                                                  # live window: CalibHessian::value_zero is not value any more
            LIB.sdv_ba_set_calib_zero.argtypes = [_vp, _f64p]; ctx._ck(LIB.sdv_ba_set_calib_zero(ctx.p, c("K_zero", np.float64)))
        ctx._ck(LIB.sdv_ba_set_points(ctx.p, self.nP, c("uv", np.float32), c("idepth", np.float32), c("idepth_zero", np.float32), c("color", np.float32),
                                      c("weights", np.float32), c("host", np.int32), c("hasDepthPrior", np.int32), c("isFromSensor", np.int32), c("res_begin", np.int32),
                                      self.nR, c("r_point", np.int32), c("r_host", np.int32), c("r_target", np.int32), c("r_hasMatcher", np.int32),
                                      c("r_matcher", np.float32), c("r_isNew", np.int32)))

    @staticmethod
    def install_batch(ctx: "Context", windows, wins, frame_ids_list):
        """EnergyFunctional(ctx, wins[i], frame_ids_list[i], window=windows[i]) for every i, in two calls (sdv_ba_set_window_batch, sdv_ba_set_points_batch)."""
        _ba_protos(); w = np.ascontiguousarray(windows, np.int32); n = len(w); k = pack_ba_windows(wins, frame_ids_list)
        ptr = lambda a: None if a is None else a.ctypes.data
        ctx._ck(LIB.sdv_ba_set_window_batch(ctx.p, n, w, k["f_begin"], k["frame_ids"], k["T_eval"], k["state"], k["state_zero"], k["ab_exposure"], k["frameID"],
                                            k["frameEnergyTH"], k["K"], ptr(k["K_zero"]), ptr(k["HM"]), ptr(k["bM"])))
        ctx._ck(LIB.sdv_ba_set_points_batch(ctx.p, n, w, k["p_begin"], k["r_begin"], k["uv"], k["idepth"], k["idepth_zero"], k["color"], k["weights"], k["host"],
                                            k["hasDepthPrior"], k["isFromSensor"], k["res_begin"], k["r_point"], k["r_host"], k["r_target"], k["r_hasMatcher"],
                                            k["r_matcher"], k["r_isNew"]))
        out = []
        for i, win in enumerate(wins):
            e = EnergyFunctional.__new__(EnergyFunctional); e.ctx = ctx; e.win = win; e.window = int(w[i])
            e.nF = int(win["nF"]); e.nP = len(win["uv"]); e.nR = len(win["r_point"]); e.n = 4 + 6 * e.nF
            out.append(e)
        return out

    def _sel(self): self.ctx._ck(LIB.sdv_ba_select(self.ctx.p, self.window))
    def reset_oob(self): self._sel(); self.ctx._ck(LIB.sdv_ba_reset_oob(self.ctx.p))
    def linearizeAll(self, fix=False):
        self._sel(); e = C.c_double(0); self.ctx._ck(LIB.sdv_ba_linearize(self.ctx.p, 1 if fix else 0, C.byref(e))); return e.value
    def applyRes(self): self._sel(); self.ctx._ck(LIB.sdv_ba_apply_res(self.ctx.p))
    def energies(self):
        self._sel(); a, b = C.c_double(0), C.c_double(0); self.ctx._ck(LIB.sdv_ba_energy(self.ctx.p, C.byref(a), C.byref(b))); return a.value, b.value
    def calcLEnergy(self): return self.energies()[0]
    def calcMEnergy(self): return self.energies()[1]
    def backupState(self): self._sel(); self.ctx._ck(LIB.sdv_ba_backup(self.ctx.p))
    def doStepFromBackup(self, f=1.0):
        self._sel(); cb = C.c_int(0); self.ctx._ck(LIB.sdv_ba_step(self.ctx.p, f, 0, C.byref(cb))); return bool(cb.value)
    def loadStateBackup(self):
        self._sel(); cb = C.c_int(0); self.ctx._ck(LIB.sdv_ba_step(self.ctx.p, 1.0, 1, C.byref(cb)))

    def solveSystem(self, iteration, lam):
        self._sel(); n = self.n; x = np.zeros(n); self.ctx._ck(LIB.sdv_ba_solve(self.ctx.p, iteration, lam, x))
        HA = np.zeros((n, n)); bA = np.zeros(n); Hsc = np.zeros((n, n)); bsc = np.zeros(n); HS = np.zeros((n, n)); bS = np.zeros(n)
        self.ctx._ck(LIB.sdv_ba_get_system(self.ctx.p, HA, bA, Hsc, bsc, HS, bS))
        return x, HS, bS, (HA, bA, Hsc, bsc)

    def optimize(self, its=6):
        self._sel(); r = C.c_float(0); i = C.c_int32(0); a = C.c_int32(0)
        self.ctx._ck(LIB.sdv_ba_optimize(self.ctx.p, its, C.byref(r), C.byref(i), C.byref(a)))
        return dict(rmse=float(r.value), iterations=int(i.value), accepts=int(a.value), ms=float(LIB.sdv_ba_last_kernel_ms(self.ctx.p)))

    def residuals(self):
        self._sel(); n = self.nR
        o = dict(state=np.zeros(n, np.int32), new_state=np.zeros(n, np.int32), energies=np.zeros((n, 3), np.float32), active=np.zeros(n, np.int32),
                 J=np.zeros((n, 24), np.float32), efJ=np.zeros((n, 24), np.float32), JpJdF=np.zeros((n, 8), np.float32),
                 center=np.zeros((n, 3), np.float32), toRemove=np.zeros(n, np.int32))
        self.ctx._ck(LIB.sdv_ba_get_residuals(self.ctx.p, o["state"], o["new_state"], o["energies"], o["active"], o["J"], o["efJ"], o["JpJdF"], o["center"], o["toRemove"]))
        return o

    def points(self):
        self._sel(); n = self.nP
        o = dict(idepth=np.zeros(n, np.float32), step=np.zeros(n, np.float32), HdiF=np.zeros(n, np.float32), bdSumF=np.zeros(n, np.float32),
                 maxRelBaseline=np.zeros(n, np.float32), numGood=np.zeros(n, np.int32), idepth_hessian=np.zeros(n, np.float32))
        self.ctx._ck(LIB.sdv_ba_get_points(self.ctx.p, o["idepth"], o["step"], o["HdiF"], o["bdSumF"], o["maxRelBaseline"], o["numGood"], o["idepth_hessian"])); return o

    def frames(self):
        self._sel(); n = self.nF
        o = dict(T_eval=np.zeros((n, 7)), state=np.zeros((n, 10)), step=np.zeros((n, 10)), frameEnergyTH=np.zeros(n, np.float32), PRE_worldToCam=np.zeros((n, 7)),
                 calib_value=np.zeros(4), calib_step=np.zeros(4))
        self.ctx._ck(LIB.sdv_ba_get_frames(self.ctx.p, o["T_eval"], o["state"], o["step"], o["frameEnergyTH"], o["PRE_worldToCam"], o["calib_value"], o["calib_step"])); return o

    # ---- keyframe hand-over (FullSystem::makeKeyFrame after optimize, FullSystem.cpp:1152-1171)
    def flagPointsForRemoval(self, selected):
        self._sel(); st = np.zeros(self.nP, np.int32)
        self.ctx._ck(LIB.sdv_ba_flag_points(self.ctx.p, np.ascontiguousarray(selected, np.int32), st)); return st

    def marginalizePointsF(self, status=None):
        self._sel(); st = None if status is None else np.ascontiguousarray(status, np.int32)
        self.ctx._ck(LIB.sdv_ba_marginalize_points(self.ctx.p, None if st is None else st.ctypes.data))
        n = self.n; M = np.zeros((n, n)); Mb = np.zeros(n); S = np.zeros((n, n)); Sb = np.zeros(n)
        d1 = np.zeros((n, n)); d2 = np.zeros(n)
        self.ctx._ck(LIB.sdv_ba_get_system(self.ctx.p, M, Mb, S, Sb, d1, d2))
        return dict(M=M, Mb=Mb, Msc=S, Mbsc=Sb)

    def marginalizeFrame(self, idx: int):
        self._sel(); self.ctx._ck(LIB.sdv_ba_marginalize_frame(self.ctx.p, int(idx)))
        self.nF -= 1; self.n -= 6; self.nP = 0; self.nR = 0

    def prior(self):
        self._sel(); d = C.c_int(0); self.ctx._ck(LIB.sdv_ba_get_prior(self.ctx.p, C.byref(d), None, None))
        n = d.value; HM = np.zeros((n, n)); bM = np.zeros(n)
        self.ctx._ck(LIB.sdv_ba_get_prior(self.ctx.p, C.byref(d), HM.ctypes.data, bM.ctypes.data)); return HM, bM

    def linearized(self):
        self._sel(); r = np.zeros((self.nR, 2), np.float32); l = np.zeros(self.nR, np.int32)
        self.ctx._ck(LIB.sdv_ba_get_linearized(self.ctx.p, r, l)); return r, l

    def precalc(self, host, target):
        self._sel(); o = np.zeros(27, np.float32); aH = np.zeros(36); aT = np.zeros(36); d = np.zeros(6, np.float32)
        self.ctx._ck(LIB.sdv_ba_get_precalc(self.ctx.p, host, target, o, aH, aT, d))
        return dict(KRKi=o[:9].reshape(3, 3), Kt=o[9:12], R0=o[12:21].reshape(3, 3), t0=o[21:24], aff=o[24:26], b0=o[26], adHost=aH.reshape(6, 6), adTarget=aT.reshape(6, 6), adHTdelta=d)


def _ba_group(efs):
    assert efs and all(e.ctx is efs[0].ctx for e in efs), "one context"
    _ba_protos(); return efs[0].ctx, np.array([e.window for e in efs], np.int32)


def flag_points_batch(efs, selected):
    """EnergyFunctional.flagPointsForRemoval of several windows in one call: selected[i] per window -> status per window"""
    ctx, w = _ba_group(efs); sel = _cat(selected, np.int32); st = np.zeros(len(sel), np.int32)
    assert len(sel) == sum(e.nP for e in efs)
    ctx._ck(LIB.sdv_ba_flag_points_batch(ctx.p, len(w), w, sel, st.ctypes.data))
    return np.split(st, np.cumsum([e.nP for e in efs])[:-1])


def marginalize_points_batch(efs, status=None):
    """EnergyFunctional.marginalizePointsF of several windows in one call (status None: the device-resident result of the flag call)"""
    ctx, w = _ba_group(efs); st = None if status is None else _cat(status, np.int32)
    ctx._ck(LIB.sdv_ba_marginalize_points_batch(ctx.p, len(w), w, None if st is None else st.ctypes.data))


def marginalize_frames_batch(efs, idx_lists, prior: bool = True):
    """EnergyFunctional.marginalizeFrame of several windows in one call: window i eliminates idx_lists[i] in order (each index into the window as the previous
    eliminations left it).  Returns each window's (HM, bM) afterwards when prior is set."""
    ctx, w = _ba_group(efs); k = np.array([len(x) for x in idx_lists], np.int64); kb = np.concatenate([[0], np.cumsum(k)]).astype(np.int32)
    idx = _cat(idx_lists, np.int32); dims = [e.n - 6 * int(kk) for e, kk in zip(efs, k)]
    HM = np.zeros(sum(d * d for d in dims)) if prior else None; bM = np.zeros(sum(dims)) if prior else None
    ctx._ck(LIB.sdv_ba_marginalize_frames_batch(ctx.p, len(w), w, kb, idx, None if HM is None else HM.ctypes.data, None if bM is None else bM.ctypes.data))
    for e, kk in zip(efs, k):
        if kk:
            e.nF -= int(kk); e.n -= 6 * int(kk); e.nP = 0; e.nR = 0
    if not prior:
        return None
    out, h, b = [], 0, 0
    for d in dims:
        out.append((HM[h:h + d * d].reshape(d, d), bM[b:b + d])); h += d * d; b += d
    return out


def optimize_batch(ctx: Context, windows, its: int = 6):
    """FullSystem::optimize on several windows of one context in one device-resident schedule."""
    _ba_protos(); w = np.ascontiguousarray(windows, np.int32); n = len(w)
    rmse = np.zeros(n, np.float32); it = np.zeros(n, np.int32); acc = np.zeros(n, np.int32)
    ctx._ck(LIB.sdv_ba_optimize_batch(ctx.p, n, w, its, rmse, it, acc))
    return dict(rmse=rmse, iterations=it, accepts=acc, ms=float(LIB.sdv_ba_last_kernel_ms(ctx.p)))


# ---------------------------------------------------------------------------------------------- immature points: ImmaturePoint ctor + traceOn (sdv_trace.cu)
IMMATURE_PT_DTYPE = np.dtype([("u", np.float32), ("v", np.float32), ("idepth_min", np.float32), ("idepth_max", np.float32), ("color", np.float32, 8), ("weights", np.float32, 8),
                              ("gradH", np.float32, 4), ("energyTH", np.float32), ("quality", np.float32), ("lastTraceUV", np.float32, 2), ("lastTracePixelInterval", np.float32),
                              ("lastTraceStatus", np.int32)])
IPS_GOOD, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED = range(6)


def immatureInit(ctx: Context, host_frame_id: int, uv, cam: int = 0):
    """ImmaturePoint::ImmaturePoint (ImmaturePoint.cpp:8-36) for integer pixels uv (n,2) of a resident keyframe of camera `cam` -> IMMATURE_PT_DTYPE array"""
    uv = np.ascontiguousarray(uv, np.int32).reshape(-1, 2); P = np.zeros(len(uv), IMMATURE_PT_DTYPE)
    if cam == 0:
        ctx._ck(LIB.sdv_immature_init(ctx.p, host_frame_id, len(uv), uv.reshape(-1), P.ctypes.data))
    else:
        ctx._ck(LIB.sdv_immature_init_cam(ctx.p, int(cam), host_frame_id, len(uv), uv.reshape(-1), P.ctypes.data))
    return P


def traceOnBatch(ctx: Context, frame_ids, pt_begin, KRKi, Kt, aff, pts, cams=None):
    """ImmaturePoint::traceOn for every candidate of every (host keyframe, traced frame) group — the loop of FullSystem::traceNewCoarse (FullSystem.cpp:519-552), batched.
    Group g traces at camera cams[g]'s size (None: camera 0).  pts (IMMATURE_PT_DTYPE) is updated in place; returns the statuses."""
    assert pts.dtype == IMMATURE_PT_DTYPE and pts.flags.c_contiguous
    ng = len(frame_ids); pb = np.ascontiguousarray(pt_begin, np.int32); assert len(pb) == ng + 1 and pb[-1] == len(pts)
    st = np.zeros(len(pts), np.int32); cm = Context._cams(cams, ng)
    args = (np.ascontiguousarray(frame_ids, np.uint64), pb, np.ascontiguousarray(KRKi, np.float32).reshape(-1), np.ascontiguousarray(Kt, np.float32).reshape(-1),
            np.ascontiguousarray(aff, np.float32).reshape(-1), pts.ctypes.data, st.ctypes.data)
    if cm is None:
        ctx._ck(LIB.sdv_immature_trace_batch(ctx.p, ng, *args))
    else:
        ctx._ck(LIB.sdv_immature_trace_batch_cams(ctx.p, ng, args[0], cm.ctypes.data, *args[1:]))
    return st


def optimizeImmaturePointBatch(ctx: Context, pt_begin, tgt_begin, target_frame_ids, pre14, calib6, pts, is_from_sensor=None, min_obs=1, cams=None):
    """FullSystem::optimizeImmaturePoint (FullSystemOptPoint.cpp:18-183) for the candidates of several host keyframes in one launch (group = host; see sdv_b200.h).
    Group g works at camera cams[g]'s size (None: camera 0); its targets must have that size.
    Returns (status (n,) 0 stay / -1 drop / 1 activate, idepth (n,), res_state (n, stride) with -1 padding)."""
    assert pts.dtype == IMMATURE_PT_DTYPE and pts.flags.c_contiguous
    pb = np.ascontiguousarray(pt_begin, np.int32); tb = np.ascontiguousarray(tgt_begin, np.int32); ng = len(pb) - 1; n = len(pts); assert pb[-1] == n and len(tb) == ng + 1
    stride = max(1, int(np.diff(tb).max())) if ng else 1
    st = np.zeros(n, np.int32); idp = np.zeros(n, np.float32); rs = np.full((n, stride), -1, np.int32)
    fs = None if is_from_sensor is None else np.ascontiguousarray(is_from_sensor, np.uint8); cm = Context._cams(cams, ng)
    head = (pb, tb, np.ascontiguousarray(target_frame_ids, np.uint64), np.ascontiguousarray(pre14, np.float32).reshape(-1), np.ascontiguousarray(calib6, np.float32).reshape(-1))
    tail = (min_obs, pts.ctypes.data, None if fs is None else fs.ctypes.data, stride, st, idp, rs.reshape(-1))
    if cm is None:
        ctx._ck(LIB.sdv_immature_optimize_batch(ctx.p, ng, *head, *tail))
    else:
        ctx._ck(LIB.sdv_immature_optimize_batch_cams(ctx.p, ng, *head, cm.ctypes.data, *tail))
    return st, idp, rs


IMMATURE_META_DTYPE = np.dtype([("my_type", np.float32), ("type", np.int32), ("isFromSensor", np.int32), ("idepth_fromSensor", np.float32)])


class ImmatureStore:
    """host->immaturePoints of every keyframe of a context, kept on the device: one block per host keyframe, keyed by its frame id (sdv_immature_store_*).
    The records never need to come back to the host: PixelSelector.makeNewTracesStore fills a block, traceStoreBatch traces blocks in place, drop forgets them."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def set(self, host_frame_id: int, pts, meta=None):
        """replace the block of host_frame_id by pts (IMMATURE_PT_DTYPE) and meta (IMMATURE_META_DTYPE; None: my_type 1, type -1, not from the sensor)"""
        p = np.ascontiguousarray(pts, IMMATURE_PT_DTYPE); m = None if meta is None else np.ascontiguousarray(meta, IMMATURE_META_DTYPE)
        assert m is None or len(m) == len(p)
        self.ctx._ck(LIB.sdv_immature_store_set(self.ctx.p, int(host_frame_id), len(p), p.ctypes.data if len(p) else None, None if m is None else m.ctypes.data))

    def count(self, host_frame_ids):
        h = np.ascontiguousarray(np.atleast_1d(host_frame_ids), np.uint64); o = np.zeros(len(h), np.int32)
        self.ctx._ck(LIB.sdv_immature_store_count(self.ctx.p, len(h), h, o)); return o

    def get(self, host_frame_id: int):
        """(records, meta) of the block of host_frame_id in its current order"""
        n = self.count([host_frame_id])[0]; P = np.zeros(n, IMMATURE_PT_DTYPE); M = np.zeros(n, IMMATURE_META_DTYPE); no = C.c_int32(0)
        self.ctx._ck(LIB.sdv_immature_store_get(self.ctx.p, int(host_frame_id), int(n), P.ctypes.data, M.ctypes.data, C.byref(no))); return P, M

    def drop(self, host_frame_ids):
        h = np.ascontiguousarray(np.atleast_1d(host_frame_ids), np.uint64); self.ctx._ck(LIB.sdv_immature_store_drop(self.ctx.p, len(h), h))


def traceStoreBatch(ctx: Context, host_frame_ids, frame_ids, KRKi, Kt, aff, cams=None, counts=False):
    """FullSystem::traceNewCoarse on the store: group g traces every point of host_frame_ids[g]'s block into frame_ids[g] (camera cams[g]; None: camera 0), in place.
    counts=True waits for the device and returns the (n, 6) per-status counts after the trace (column s: lastTraceStatus == s); else returns None at once."""
    ng = len(host_frame_ids); cm = Context._cams(cams, ng); co = np.zeros((ng, 6), np.int32) if counts else None
    ctx._ck(LIB.sdv_immature_trace_store_batch(ctx.p, ng, np.ascontiguousarray(host_frame_ids, np.uint64), np.ascontiguousarray(frame_ids, np.uint64), None if cm is None else cm.ctypes.data,
                                               np.ascontiguousarray(KRKi, np.float32).reshape(-1), np.ascontiguousarray(Kt, np.float32).reshape(-1),
                                               np.ascontiguousarray(aff, np.float32).reshape(-1), None if co is None else co.ctypes.data))
    return co


def activateStoreBatch(ctx: Context, seqs, cams=None, cap=1 << 16):
    """FullSystem::activatePointsMT (FullSystem.cpp:598-720) on the ImmatureStore for several sequences.  seqs: dicts with hosts (window keyframe ids, newest last), flagged,
    cKRKi / cKt (per host), the distance-map sources pt_begin / KRKi / Kt / uvid as activateSelectBatch takes them, minActDist, pre14 ((host, target) rows, host-major,
    targets = the window without the host), calib6.  -> dict of per-sequence lists: host (index into the sequence's hosts), idx, pts, meta, idepth, res_state (k, nH-1),
    and counts (block sizes after the compaction)"""
    f = lambda a, t: np.ascontiguousarray(a, t); n = len(seqs); P = packActivation(seqs, cams)
    hb = f(np.concatenate([[0], np.cumsum([len(q["hosts"]) for q in seqs])]), np.int32); NH = int(hb[-1])
    hosts = f(np.concatenate([q["hosts"] for q in seqs]), np.uint64); fl = f(np.concatenate([q["flagged"] for q in seqs]), np.int32)
    cA = f(np.concatenate([np.asarray(q["cKRKi"], np.float32).reshape(-1, 9) for q in seqs]), np.float32); cB = f(np.concatenate([np.asarray(q["cKt"], np.float32).reshape(-1, 3) for q in seqs]), np.float32)
    pre = f(np.concatenate([np.asarray(q["pre14"], np.float32).reshape(-1, 14) for q in seqs] + [np.zeros((1, 14), np.float32)]), np.float32)
    cal = f(np.stack([np.asarray(q["calib6"], np.float32) for q in seqs]), np.float32); R = 8
    n_act = np.zeros(n, np.int32); ah = np.zeros(cap, np.int32); ai = np.zeros(cap, np.int32); ap = np.zeros(cap, IMMATURE_PT_DTYPE); am = np.zeros(cap, IMMATURE_META_DTYPE)
    aid = np.zeros(cap, np.float32); ars = np.zeros((cap, R), np.int32); cnt = np.zeros(NH, np.int32); cm = P["cams"]
    ctx._ck(LIB.sdv_activate_points_store_batch(ctx.p, n, hb, hosts, fl, cA, cB, P["hb"], P["pb"], P["A"].ctypes.data, P["B"].ctypes.data, P["U"].ctypes.data, P["md"], pre, cal,
                                                None if cm is None else cm.ctypes.data, cap, n_act, ah.ctypes.data, ai.ctypes.data, ap.ctypes.data, am.ctypes.data, aid.ctypes.data,
                                                ars.ctypes.data, cnt.ctypes.data))
    out = dict(host=[], idx=[], pts=[], meta=[], idepth=[], res_state=[], counts=[]); o = 0
    for j in range(n):
        a = slice(o, o + n_act[j]); o += n_act[j]; nH = len(seqs[j]["hosts"])
        out["host"].append(ah[a] - hb[j]); out["idx"].append(ai[a].copy()); out["pts"].append(ap[a].copy()); out["meta"].append(am[a].copy())
        out["idepth"].append(aid[a].copy()); out["res_state"].append(ars[a, :nH - 1].copy()); out["counts"].append(cnt[hb[j]:hb[j + 1]].copy())
    return out


def coarseTrackingLogLine(frame_id: int, timestamp: float, ab_exposure: float, result: dict) -> str:
    """One line of the reference's coarseTrackingLog (FullSystem.cpp:500-513, written when setting_logStuff is on):
    id timestamp ab_exposure camToWorld.log()[6] a b achievedRes[0] tryIterations — `result` is one element of trackNewCoarseBatch's return."""
    from . import synth
    lg = synth.se3_log7(np.asarray(result["camToWorld"], np.float64))
    vals = [frame_id, timestamp, ab_exposure, *lg, result["aff_g2l"][0], result["aff_g2l"][1], result["lastCoarseRMSE"][0], result["tries"]]
    return " ".join(("%d" % v) if isinstance(v, (int, np.integer)) else ("%.16g" % v) for v in vals)


# ---------------------------------------------------------------------------------------------- candidate management at keyframe rate (sdv_select.cu)
NEW_TRACE_DTYPE = np.dtype([("u", "<f4"), ("v", "<f4"), ("my_type", "<f4"), ("score", "<f4"), ("idepth_fromSensor", "<f4"), ("isFromSensor", "<i4"), ("type", "<i4")])


def random_pattern(w: int, h: int):
    """PixelSelector::randomPattern (PixelSelector2.cpp:14-16): srand(3141592); rand() & 0xFF, w*h times — the C library's generator, like the reference.
    NB: re-seeds the process-wide rand() stream exactly as constructing a PixelSelector does."""
    libc = C.CDLL(None); libc.srand(3141592)
    return np.array([libc.rand() & 0xFF for _ in range(w * h)], np.uint8)


def initializer_draws(w: int, h: int, n: int, seed: int = 3141592):
    """the n rand() values FullSystem::initializeFromInitializer draws in a running reference (FullSystem.cpp:1203): the frame-0 PixelSelector re-seeds the C library
    (srand(3141592)) and draws w*h values for its pattern, nothing else calls rand() before.  NB: re-seeds the process-wide rand() stream, like random_pattern."""
    libc = C.CDLL(None); libc.srand(seed)
    for _ in range(w * h):
        libc.rand()
    return np.array([libc.rand() for _ in range(n)], np.int32)


def initializeFromLidarBatch(ctx: "Context", slots, frame_ids, clouds, lruds, desired_point_density, draws, cap: int = 1 << 14):
    """The start of n sequences (sdv_init_from_lidar_batch / _rows_batch): CoarseInitializer::setFirstFromLidar at level 0 on keyframe frame_ids[j], the point loop of
    FullSystem::initializeFromInitializer with job j's rand() values draws[j] (at least one per row), and setCTRefForFirstFrame + the one-keyframe map installed on
    tracker / map slot slots[j].  clouds (n arrays of rows {Ku, Kv, depth}) and lruds (n boxes) given: the host form; None: the rows and box of each frame's LiDAR row
    set.  -> dict(pts, meta, idepth: per-job record arrays of the kept points, n_selected = numPoints[0] per job (the rand() draws consumed), n = points kept)"""
    n = len(slots); sl = np.ascontiguousarray(slots, np.int32); fr = np.ascontiguousarray(frame_ids, np.uint64)
    dens = np.ascontiguousarray(np.broadcast_to(desired_point_density, n), np.float32)
    dr = [np.ascontiguousarray(d, np.int32).reshape(-1) for d in draws]; db = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(d) for d in dr])]), np.int32)
    da = np.ascontiguousarray(np.concatenate(dr) if sum(len(d) for d in dr) else np.zeros(1), np.int32)
    n_out = np.zeros(n, np.int32); n_sel = np.zeros(n, np.int32)
    P = np.zeros((n, max(cap, 1)), IMMATURE_PT_DTYPE); M = np.zeros((n, max(cap, 1)), IMMATURE_META_DTYPE); D = np.zeros((n, max(cap, 1)), np.float32)
    if clouds is None:
        ctx._ck(LIB.sdv_init_from_lidar_rows_batch(ctx.p, n, sl, fr, dens, db, da, cap, n_out, n_sel, P.ctypes.data, M.ctypes.data, D.ctypes.data))
    else:
        cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; cb = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(c) for c in cl])]), np.int32)
        c3 = np.ascontiguousarray(np.concatenate(cl) if cb[-1] else np.zeros((1, 3)), np.float64); box = np.ascontiguousarray(lruds, np.int32).reshape(n * 4)
        ctx._ck(LIB.sdv_init_from_lidar_batch(ctx.p, n, sl, fr, cb, c3.ctypes.data, box, dens, db, da, cap, n_out, n_sel, P.ctypes.data, M.ctypes.data, D.ctypes.data))
    return dict(pts=[P[j, :n_out[j]].copy() for j in range(n)], meta=[M[j, :n_out[j]].copy() for j in range(n)], idepth=[D[j, :n_out[j]].copy() for j in range(n)],
                n_selected=n_sel, n=n_out)


def lidar_density(lrud, wh, desiredImmatureDensity):
    """((float)lidarArea/(float)imageArea) * setting_desiredImmatureDensity with lidarArea = (right-left)*(down-up)   FullSystem.cpp:1287-1290"""
    area = (lrud[1] - lrud[0]) * (lrud[3] - lrud[2])
    return float(np.float32(np.float32(area) / np.float32(wh[0] * wh[1])) * np.float32(desiredImmatureDensity))


class PixelSelector:
    """n_slots PixelSelector + selectionMap pairs (one per resident sequence) of a context: FullSystem/PixelSelector2.cpp, FullSystem.cpp:180-186.
    Slot s works at its camera's size (cams[s], bindCams; camera 0 by default): its frames, its selection map."""

    def __init__(self, ctx: Context, n_slots: int = 1, pattern=None, cams=None):
        self.ctx = ctx; self.n_slots = n_slots; self.slot_cam = {}       # slot -> camera, for slots not on camera 0
        self.pattern = np.ascontiguousarray(pattern if pattern is not None else random_pattern(ctx.w, ctx.h), np.uint8); assert self.pattern.size == ctx.w * ctx.h
        ctx._ck(LIB.sdv_selector_init(ctx.p, self.pattern.ctypes.data, n_slots))
        if cams is not None:
            self.bindCams(range(n_slots), cams)

    def bindCams(self, slots, cams):
        """slot slots[i] works at camera cams[i]'s size from now on; moving it to a camera of another size starts it afresh (a new PixelSelector and selectionMap)"""
        sl = np.ascontiguousarray(list(slots), np.int32).reshape(-1); cm = Context._cams(cams, len(sl))
        self.ctx._ck(LIB.sdv_selector_set_slot_cams(self.ctx.p, len(sl), sl, cm))
        for s, c in zip(sl.tolist(), cm.tolist()):
            if c:
                self.slot_cam[s] = c
            else:
                self.slot_cam.pop(s, None)

    def slotSize(self, slot):
        return self.ctx.camSize(self.slot_cam.get(int(slot), 0))

    def potential(self, slot=0, set_to=None) -> int:
        o = C.c_int(0); self.ctx._ck(LIB.sdv_selector_potential(self.ctx.p, slot, int(set_to) if set_to else 0, C.byref(o))); return o.value

    def selectionMap(self, slot=0):
        w, h = self.slotSize(slot); o = np.zeros((h, w), np.uint8); self.ctx._ck(LIB.sdv_selector_get_map(self.ctx.p, slot, o.ctypes.data)); return o

    def makeHists(self, frame_id, cam: int = 0):
        w, h = self.ctx.camSize(cam); n = (w // 32) * (h // 32); a = np.zeros(n, np.float32); b = np.zeros(n, np.float32)
        self.ctx._ck(LIB.sdv_selector_make_hists_cam(self.ctx.p, int(cam), frame_id, a.ctypes.data, b.ctypes.data)); return a, b

    def makeMapsBatch(self, slots, frame_ids, density, recursionsLeft=1, thFactor=1.0, clouds=None):
        """makeMapsFromLidar (clouds: one (n,3) float64 array {Ku,Kv,depth} per job) or makeMaps (clouds None) for several (slot, frame) pairs -> maps, numHaveSub.
        makeMaps returns an (n, h, w) array when every slot has the context size, else a list of per-job (h_c, w_c) maps."""
        n = len(slots); sl = np.ascontiguousarray(slots, np.int32); fr = np.ascontiguousarray(frame_ids, np.uint64)
        de = np.ascontiguousarray(np.broadcast_to(density, n), np.float32); rc = np.ascontiguousarray(np.broadcast_to(recursionsLeft, n), np.int32); th = np.ascontiguousarray(np.broadcast_to(thFactor, n), np.float32)
        num = np.zeros(n, np.int32)
        if clouds is None:
            whs = [self.slotSize(s) for s in sl.tolist()]
            if all(wh == (self.ctx.w, self.ctx.h) for wh in whs):
                maps = np.zeros((n, self.ctx.h, self.ctx.w), np.uint8)
                self.ctx._ck(LIB.sdv_selector_make_maps_batch(self.ctx.p, n, sl, fr, None, None, de, rc, th, maps.ctypes.data, num)); return maps, num
            off = np.concatenate([[0], np.cumsum([w * h for w, h in whs])]); flat = np.zeros(int(off[-1]), np.uint8)
            self.ctx._ck(LIB.sdv_selector_make_maps_batch(self.ctx.p, n, sl, fr, None, None, de, rc, th, flat.ctypes.data, num))
            return [flat[off[j]:off[j + 1]].reshape(whs[j][1], whs[j][0]) for j in range(n)], num
        cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; cb = np.concatenate([[0], np.cumsum([len(c) for c in cl])]).astype(np.int32)
        allc = np.ascontiguousarray(np.concatenate(cl) if cb[-1] else np.zeros((1, 3))); maps = np.zeros(max(int(cb[-1]), 1), np.uint8)
        self.ctx._ck(LIB.sdv_selector_make_maps_batch(self.ctx.p, n, sl, fr, cb.ctypes.data, allc.ctypes.data, de, rc, th, maps.ctypes.data, num))
        return [maps[cb[j]:cb[j + 1]] for j in range(n)], num

    def makeNewTracesBatch(self, slots, frame_ids, clouds, density_lidar, density_dense, add_feature_point, cap=1 << 14):
        """FullSystem::makeNewTraces for one new keyframe per slot -> per job (sdv_new_trace records, sdv_immature_pt records), numPoints (n,2)"""
        cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; cb = np.concatenate([[0], np.cumsum([len(c) for c in cl])]).astype(np.int32)
        allc = np.ascontiguousarray(np.concatenate(cl) if cb[-1] else np.zeros((1, 3)))
        res, num = self.makeNewTracesPacked(slots, frame_ids, allc, cb, density_lidar, density_dense, add_feature_point, cap)
        return [(t.copy(), i.copy()) for t, i in res], num

    def makeNewTracesPacked(self, slots, frame_ids, cloud_all, cloud_begin, density_lidar, density_dense, add_feature_point, cap=1 << 14):
        """the same with the pixel rows of all jobs already back to back in ONE float64 (N,3) host array and their row offsets; the returned record arrays are VIEWS into
        buffers this object reuses (valid until the next call) — nothing is copied or zeroed on the host"""
        n = len(slots); cb = np.ascontiguousarray(cloud_begin, np.int32); assert cloud_all.dtype == np.float64 and cloud_all.flags.c_contiguous and len(cb) == n + 1
        if getattr(self, "_nt_buf", None) is None or self._nt_buf[0].shape != (n, cap):
            self._nt_buf = (np.empty((n, cap), NEW_TRACE_DTYPE), np.empty((n, cap), IMMATURE_PT_DTYPE))
        out, imm = self._nt_buf; n_out = np.zeros(n, np.int32); num = np.zeros(2 * n, np.int32)
        self.ctx._ck(LIB.sdv_make_new_traces_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frame_ids, np.uint64), cb, cloud_all.ctypes.data,
                                                  np.ascontiguousarray(np.broadcast_to(density_lidar, n), np.float32), np.ascontiguousarray(np.broadcast_to(density_dense, n), np.float32),
                                                  np.ascontiguousarray(np.broadcast_to(add_feature_point, n), np.int32), cap, out.ctypes.data, imm.ctypes.data, n_out, num))
        return [(out[j, :n_out[j]], imm[j, :n_out[j]]) for j in range(n)], num.reshape(n, 2)

    def makeNewTracesStore(self, slots, frame_ids, clouds, density_lidar, density_dense, add_feature_point, cap=1 << 14):
        """FullSystem::makeNewTraces for one new keyframe per slot, the points deposited into the ImmatureStore block of frame_ids[j] (sensor points with their LiDAR
        depth and status SKIPPED, as makeNewTraces / makeKeyFrame leave them) -> points per job (n,), numPoints (n,2)"""
        n = len(slots); cl = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]; cb = np.concatenate([[0], np.cumsum([len(c) for c in cl])]).astype(np.int32)
        allc = np.ascontiguousarray(np.concatenate(cl) if cb[-1] else np.zeros((1, 3))); n_out = np.zeros(n, np.int32); num = np.zeros(2 * n, np.int32)
        self.ctx._ck(LIB.sdv_make_new_traces_store_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frame_ids, np.uint64), cb, allc.ctypes.data,
                                                        np.ascontiguousarray(np.broadcast_to(density_lidar, n), np.float32), np.ascontiguousarray(np.broadcast_to(density_dense, n), np.float32),
                                                        np.ascontiguousarray(np.broadcast_to(add_feature_point, n), np.int32), cap, n_out, num))
        return n_out, num.reshape(n, 2)

    def lidarBox(self, slot=0, set_to=None):
        """FullSystem::left, right, up, down of the sequence on `slot` (set_to: write it first, e.g. for a start in mid-drive) -> int32 (4,)"""
        o = np.zeros(4, np.int32); st = None if set_to is None else np.ascontiguousarray(set_to, np.int32).reshape(4)
        self.ctx._ck(LIB.sdv_selector_lidar_box(self.ctx.p, int(slot), None if st is None else st.ctypes.data, o.ctypes.data)); return o

    def makeNewTracesRowsStore(self, slots, frame_ids, desired_density, cap=1 << 14):
        """makeNewTracesStore fed from the LiDAR row sets of frame_ids (LidarFrontEnd.handleRows): rows, box and addFeaturePoint of each frame's set, which never come
        to the host; density_lidar follows from the set's box and the slot's camera size -> points per job (n,), numPoints (n,2)"""
        n = len(slots); n_out = np.zeros(n, np.int32); num = np.zeros(2 * n, np.int32)
        self.ctx._ck(LIB.sdv_make_new_traces_rows_store_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frame_ids, np.uint64),
                                                             np.ascontiguousarray(np.broadcast_to(desired_density, n), np.float32), cap, n_out, num))
        return n_out, num.reshape(n, 2)


def packActivation(seqs, cams=None):
    """the flat arrays sdv_activate_select_batch(_cams) takes, from per-sequence dicts with pt_begin / KRKi / Kt / uvid (source keyframes) and cand_begin / cKRKi / cKt / cand4 /
    minActDist (candidate keyframes; may be absent); cams: the camera of each sequence (None: camera 0)"""
    hb, pb, gb, cb = [0], [0], [0], [0]; A, B, U, cA, cB, c4, md = [], [], [], [], [], [], []
    f = lambda a, t: np.ascontiguousarray(a, t)
    for q in seqs:
        p = f(q["pt_begin"], np.int32); hb.append(hb[-1] + len(p) - 1); pb += list(pb[-1] + p[1:]); A.append(f(q["KRKi"], np.float32).reshape(-1, 9)); B.append(f(q["Kt"], np.float32).reshape(-1, 3)); U.append(f(q["uvid"], np.float32).reshape(-1, 3))
        g = f(q.get("cand_begin", [0]), np.int32); gb.append(gb[-1] + len(g) - 1); cb += list(cb[-1] + g[1:]); md.append(q.get("minActDist", 0.0))
        if len(g) > 1: cA.append(f(q["cKRKi"], np.float32).reshape(-1, 9)); cB.append(f(q["cKt"], np.float32).reshape(-1, 3)); c4.append(f(q["cand4"], np.float32).reshape(-1, 4))
    cat = lambda xs, k: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros((1, k), np.float32))
    return dict(n=len(seqs), hb=f(hb, np.int32), pb=f(pb, np.int32), A=cat(A, 9), B=cat(B, 3), U=cat(U, 3), gb=f(gb, np.int32), cb=f(cb, np.int32), cA=cat(cA, 9), cB=cat(cB, 3), c4=cat(c4, 4),
                md=f(md, np.float32), dec=np.zeros(max(cb[-1], 1), np.int32), cams=Context._cams(cams, len(seqs)))


def activateSelectPacked(ctx: Context, P, want_maps=False):
    """sdv_activate_select_batch on arrays packed by packActivation (the decisions land in P['dec'], reused between calls) -> per-sequence views of the decisions (+ maps:
    an (n, h/2, w/2) array when the sequences are on camera 0, else a list of per-sequence level-1 maps at each camera's size)"""
    n = P["n"]; cm = P.get("cams"); maps = None
    if cm is None:
        maps = np.zeros((n, ctx.h >> 1, ctx.w >> 1), np.float32) if want_maps else None; flat = maps
    elif want_maps:
        whs = [ctx.camSize(c) for c in cm.tolist()]; off = np.concatenate([[0], np.cumsum([(w >> 1) * (h >> 1) for w, h in whs])]); flat = np.zeros(int(off[-1]), np.float32)
        maps = [flat[off[j]:off[j + 1]].reshape(whs[j][1] >> 1, whs[j][0] >> 1) for j in range(n)]
    args = (P["hb"], P["pb"], P["A"].ctypes.data, P["B"].ctypes.data, P["U"].ctypes.data, P["gb"], P["cb"], P["cA"].ctypes.data, P["cB"].ctypes.data, P["c4"].ctypes.data, P["md"])
    if cm is None:
        ctx._ck(LIB.sdv_activate_select_batch(ctx.p, n, *args, P["dec"].ctypes.data, flat.ctypes.data if want_maps else None))
    else:
        ctx._ck(LIB.sdv_activate_select_batch_cams(ctx.p, n, *args, cm.ctypes.data, P["dec"].ctypes.data, flat.ctypes.data if want_maps else None))
    cb, gb = P["cb"], P["gb"]; out = [P["dec"][cb[gb[j]]:cb[gb[j + 1]]] for j in range(n)]
    return (out, maps) if want_maps else out


def activateSelectBatch(ctx: Context, seqs, want_maps=False, cams=None):
    """CoarseDistanceMap::makeDistanceMap + the candidate walk of FullSystem::activatePointsMT for several sequences.  seqs: list of dicts with pt_begin / KRKi / Kt / uvid
    (source keyframes) and cand_begin / cKRKi / cKt / cand4 / minActDist (candidate keyframes; may be absent); cams: each sequence's camera (None: camera 0).
    -> per sequence decisions (+ distance maps)"""
    r = activateSelectPacked(ctx, packActivation(seqs, cams), want_maps)
    return ([d.copy() for d in r[0]], r[1]) if want_maps else [d.copy() for d in r]


# ---------------------------------------------------------------------------------------------- LiDAR front-end (sdv_lidar.cu): lidarCloudHandler, src/main.cpp:785-858
class LidarFrontEnd:
    """projectPointCloud -> groundRemoval -> cloudSegmentation -> projection into the image, for a batch of raw XYZI sweeps (one per sequence)"""

    def __init__(self, ctx: Context, n_scan=64, horizon=1800, ang_res_x=0.2, ang_res_y=0.427, ang_bottom=24.9, groundScanInd=50):
        self.ctx = ctx; self.n_scan, self.horizon = n_scan, horizon
        ctx._ck(LIB.sdv_lidar_init(ctx.p, n_scan, horizon, ang_res_x, ang_res_y, ang_bottom, groundScanInd))

    def handle(self, sweeps, Rlc, tlc, K4, lruds, cap=None, cams=None):
        """sweeps: list of (n,4) float32 XYZI arrays; Rlc (3,3) / tlc (3,) / K4 shared or per sweep; lruds (n,4) running pixel boxes; cams: the camera of each sweep,
        whose size bounds its pixel box (None: camera 0) -> list of dicts like the oracle's"""
        sw = [np.ascontiguousarray(s, np.float32).reshape(-1, 4) for s in sweeps]; sb = np.concatenate([[0], np.cumsum([len(s) for s in sw])]).astype(np.int32)
        allp = np.ascontiguousarray(np.concatenate(sw) if sb[-1] else np.zeros((1, 4), np.float32))
        return self.handle_packed(allp, sb, Rlc, tlc, K4, lruds, cap, cams)

    def handle_packed(self, xyzi_all, sweep_begin, Rlc, tlc, K4, lruds, cap=None, cams=None):
        """the same with the sweeps already back to back in ONE host buffer (pinned or not) and their row offsets: nothing is copied on the host"""
        sb = np.ascontiguousarray(sweep_begin, np.int32); n = len(sb) - 1; allp = xyzi_all; assert allp.dtype == np.float32 and allp.flags.c_contiguous
        cap = cap or self.n_scan * self.horizon
        R = np.ascontiguousarray(np.broadcast_to(np.asarray(Rlc, np.float64).reshape(-1, 9), (n, 9))).reshape(-1); t = np.ascontiguousarray(np.broadcast_to(np.asarray(tlc, np.float64).reshape(-1, 3), (n, 3))).reshape(-1)
        K = np.ascontiguousarray(np.broadcast_to(np.asarray(K4, np.float32).reshape(-1, 4), (n, 4))).reshape(-1); lr = np.ascontiguousarray(lruds, np.int32).reshape(n, 4).copy()
        if getattr(self, "_out", None) is None or self._out.shape != (n, cap, 3): self._out = np.zeros((n, cap, 3))
        out = self._out; n_out = np.zeros(n, np.int32); add = np.zeros(n, np.int32); st = np.zeros(2 * n, np.int32)
        cm = Context._cams(cams, n)
        if cm is None:
            self.ctx._ck(LIB.sdv_lidar_handler_batch(self.ctx.p, n, sb, allp.ctypes.data, R, t, K, lr.reshape(-1), cap, out.ctypes.data, n_out, add, st))
        else:
            self.ctx._ck(LIB.sdv_lidar_handler_batch_cams(self.ctx.p, n, sb, allp.ctypes.data, R, t, K, cm.ctypes.data, lr.reshape(-1), cap, out.ctypes.data, n_out, add, st))
        return [dict(cloud_px=out[j, :n_out[j]].copy(), lrud=lr[j], numGround=int(st[2 * j]), n_segmented=int(st[2 * j + 1]), addFeaturePoint=int(add[j])) for j in range(n)]

    def handleRows(self, slots, frame_ids, sweeps, Rlc, tlc, K4, cap=None, stats=False, sweep_begin=None):
        """the handler writing into row sets (FullSystem::qCloudPixel on the device): sweep j belongs to the sequence on selector slot slots[j] (its camera, its pixel box),
        its rows go into frame_ids[j]'s set.  sweeps: list of (n,4) float32 XYZI arrays, or with sweep_begin ONE packed host buffer (pinned or not: pinned memory must stay
        valid until the next call that synchronises).  stats=False: enqueue and return None; True: wait -> per sweep dict rows, numGround, n_segmented,
        addFeaturePoint, overflow"""
        if sweep_begin is None:
            sw = [np.ascontiguousarray(s, np.float32).reshape(-1, 4) for s in sweeps]; sb = np.concatenate([[0], np.cumsum([len(s) for s in sw])]).astype(np.int32)
            allp = np.ascontiguousarray(np.concatenate(sw) if sb[-1] else np.zeros((1, 4), np.float32))
        else:
            sb = np.ascontiguousarray(sweep_begin, np.int32); allp = sweeps; assert allp.dtype == np.float32 and allp.flags.c_contiguous
        n = len(sb) - 1; cap = cap or self.n_scan * self.horizon
        R = np.ascontiguousarray(np.broadcast_to(np.asarray(Rlc, np.float64).reshape(-1, 9), (n, 9))).reshape(-1); t = np.ascontiguousarray(np.broadcast_to(np.asarray(tlc, np.float64).reshape(-1, 3), (n, 3))).reshape(-1)
        K = np.ascontiguousarray(np.broadcast_to(np.asarray(K4, np.float32).reshape(-1, 4), (n, 4))).reshape(-1); st = np.zeros((n, 5), np.int32) if stats else None
        self.ctx._ck(LIB.sdv_lidar_handler_rows_batch(self.ctx.p, n, np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frame_ids, np.uint64), sb, allp.ctypes.data, R, t, K, cap,
                                                      None if st is None else st.ctypes.data))
        if st is None:
            return None
        return [dict(rows=int(r[0]), numGround=int(r[1]), n_segmented=int(r[2]), addFeaturePoint=int(r[3]), overflow=int(r[4])) for r in st]

    def rows(self, frame_id):
        """frame_id's row set -> dict like handle()'s: cloud_px (the rows), lrud (the box after its sweep), addFeaturePoint"""
        n = C.c_int32(0); add = C.c_int32(0); lr = np.zeros(4, np.int32)
        self.ctx._ck(LIB.sdv_lidar_rows_get(self.ctx.p, int(frame_id), 0, None, C.byref(n), lr.ctypes.data, C.byref(add)))
        out = np.zeros((n.value, 3))
        if n.value:
            self.ctx._ck(LIB.sdv_lidar_rows_get(self.ctx.p, int(frame_id), n.value, out.ctypes.data, C.byref(n), None, None))
        return dict(cloud_px=out, lrud=lr, addFeaturePoint=int(add.value))

    def dropRows(self, frame_ids):
        """qCloudPixel.pop() for frame_ids (main.cpp:507)"""
        f = np.ascontiguousarray(np.atleast_1d(frame_ids), np.uint64); self.ctx._ck(LIB.sdv_lidar_rows_drop(self.ctx.p, len(f), f))
