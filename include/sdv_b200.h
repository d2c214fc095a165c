/* sdv_b200.h — C-ABI of the H100-native SDV-LOAM tracking / optimisation hot path.
 *
 * The reference (ZikangYuan/SDV-LOAM) has NO plugin/FFI layer (SURVEY.md §0 D5): the hot path sits behind C++ member
 * functions called by FullSystem.  Each entry point below names the reference member it replaces (file:line relative
 * to /root/reference/src); INTEGRATION.md shows the shim classes a maintainer adds to keep those signatures.
 *
 * Conventions
 *   - return 0 on success, negative sdv_status on error; never throws; sdv_last_error() gives the message.
 *   - NaN/inf in energies propagate unchanged (the reference signals tracking loss through them,
 *     FullSystem.cpp:862-867, FullSystemOptimize.cpp:472-476).
 *   - all pointers are HOST pointers owned by the caller and are consumed before the call returns, except the
 *     `_dev` variants which take device pointers of the context's device.
 *   - poses: double T[7] = {qw,qx,qy,qz, tx,ty,tz} (Sophus SE3d storage order, unit quaternion).
 *   - a context is bound to one CUDA device; calls on one context must not overlap (one FullSystem = one context;
 *     the reference serialises the same calls under trackMutex / mapMutex, FullSystem.h:277-323).
 */
#ifndef SDV_B200_H
#define SDV_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SDV_PYR_LEVELS 6            /* util/settings.h:25 PYR_LEVELS */
#define SDV_MAX_FRAMES_WINDOW 8     /* setting_maxFrames=7 (settings.cpp:56); 8 for the stress config */

typedef enum {
  SDV_OK = 0, SDV_ERR_ARG = -1, SDV_ERR_CUDA = -2, SDV_ERR_NOFRAME = -3, SDV_ERR_CAPACITY = -4, SDV_ERR_STATE = -5
} sdv_status;

typedef struct sdv_ctx sdv_ctx;

typedef struct { float fx, fy, cx, cy; } sdv_calib;          /* CalibHessian::value_scaledf, HessianBlocks.h:260-358 */

typedef struct {                                             /* util/settings.cpp globals that reach the hot path */
  float huberTH;                /* setting_huberTH = 6            settings.cpp:101 */
  float coarseCutoffTH;         /* setting_coarseCutoffTH = 20    settings.cpp:112 */
  float affineOptModeA;         /* <0 fix, >=0 optimise           settings.cpp:93 ; mode=1 -> 0 (main.cpp:453) */
  float affineOptModeB;         /*                                settings.cpp:94 ; mode=1 -> 0 (main.cpp:454) */
  float outlierTH;              /* setting_outlierTH = 144        settings.cpp:64 */
  float outlierTHSumComponent;  /* = 2500                         settings.cpp:65 */
  float idepthFixPrior;         /* = 2500                         settings.cpp */
  int   max_ref_points;         /* capacity of a tracker reference cloud per level (0 = w*h) */
  int   n_tracker_slots;        /* reference uses 2 (coarseTracker, coarseTracker_forNewKF; FullSystem.h); batched mode: 2 x sequences */
  int   max_frames;             /* device-resident frame pyramids kept alive at once */
  int   cluster_size;           /* CTAs per thread-block cluster per trackNewestCoarse call in the device-resident LM kernel
                                   (default 1 = batched-throughput mode; 8..16 = low-latency single-sequence mode) */
  int   track_threads;          /* threads per CTA of that kernel: 128 (default, 4 jobs resident per SM), 64 or 256 */
  int   max_kf_images;          /* pool of packed level-0 {I,dx,dy} images, built on demand for keyframes entering the BA window
                                   (0 = SDV_MAX_FRAMES_WINDOW + 4); tracked-only frames never materialise them */
} sdv_settings;

void sdv_default_settings(sdv_settings* s);

/* one per FullSystem (or one per GPU in batched mode) */
int  sdv_create(const sdv_calib* K, int w, int h, int levels, const sdv_settings* s, int device, sdv_ctx** out);
void sdv_destroy(sdv_ctx* c);
const char* sdv_last_error(sdv_ctx* c);
int  sdv_pyr_levels(int w, int h);                           /* pyrLevelsUsed rule, util/globalCalib.cpp:22-30 */
int  sdv_sync(sdv_ctx* c);                                   /* drain the context's stream */

/* Threading (SURVEY §8b): a context may be used by TWO host threads at once, split the way the reference splits its work — every sdv_ba_* entry (mapping
 * thread, FullSystem::mapMutex) on one side, every other entry (tracking thread, trackMutex) on the other.  Each side is serialised internally and runs on its own
 * stream; calls of the same side from several threads are serialised by the library. */
/* CoarseTracker::makeK(CalibHessian*) (CoarseTracker.cpp:77-106) and the CalibHessian Reprojector::reprojectMap reads (Reprojector.cpp:117-124): the bundle
 * adjustment optimises the intrinsics at every keyframe, and setCoarseTrackingRef re-derives the tracker's per-level K from them.  Replaces the context
 * calibration given to sdv_create: the default K of every later tracker / reprojection / structPoseEstimation call on a slot that has no K of its own
 * (sdv_set_calib_slots; the BA windows carry their own: sdv_ba_set_window).  Stream-ordered after the work already enqueued. */
int  sdv_set_calib(sdv_ctx* c, const sdv_calib* K);
/* CoarseTracker::makeK(CalibHessian*) per tracker instance (CoarseTracker.cpp:77-106): slot slots[i] uses K[i] from now on, for its tracker (calc_res, track,
 * track_batch, the trackNewCoarse policy) and for the map slot of the same index (reprojection, structPoseEstimation, refine).  One context can so hold
 * sequences of different cameras (of the context's size; sdv_set_calib_slots_cams for other sizes) and follow each sequence's bundle adjustment.  K == NULL: those slots follow the context
 * calibration again.  A slot's own K is kept across sdv_set_calib, sdv_tracker_set_ref, sdv_map_set and sdv_map_clear.  All-or-nothing: a bad slot or K
 * (fx, fy <= 0 or not finite; cx, cy not finite) returns SDV_ERR_ARG and changes no slot.  Stream-ordered after the work already enqueued, like sdv_set_calib. */
int  sdv_set_calib_slots(sdv_ctx* c, int n, const int32_t* slots, const sdv_calib* K);
/* The same, binding slot slots[i] (tracker and map slot) to camera cams[i] as well: its geometry row is built at that camera's rectified size
 * (sdv_set_camera_size), and every frame it reads must have that size.  cams == NULL is sdv_set_calib_slots (camera 0).  K == NULL with a camera
 * other than 0, or a camera index outside [0, SDV_MAX_CAMERAS), returns SDV_ERR_ARG (the context calibration has the context size).  Moving a slot
 * to a camera of another size while it holds a tracker reference (sdv_tracker_set_ref / _set_cloud) or a resident map (sdv_map_set, until
 * sdv_map_clear) returns SDV_ERR_STATE: those hold frames of its current size.  So the per-keyframe makeK of a slot on camera c passes cams = {c}
 * (sdv_set_calib_slots would move it back to camera 0 and is refused once the slot is in use).  All-or-nothing. */
int  sdv_set_calib_slots_cams(sdv_ctx* c, int n, const int32_t* slots, const sdv_calib* K, const int32_t* cams);

/* ---- frames: FrameHessian::makeImages(float* color, CalibHessian*)  FullSystem/HessianBlocks.cpp:107-167 ------------
 * builds the pyramid on the device, keyed by a caller-chosen handle: level 0 is kept as the planar intensity image (its {dx,dy} are
 * formed on the fly, bit-identically, by the tracker; packed level-0 texels are built lazily when the frame enters a BA window),
 * levels >= 1 as packed {I,dx,dy,absSquaredGrad} texels. */
int  sdv_frame_upload(sdv_ctx* c, uint64_t frame, const float* img_wh, float exposure);
int  sdv_frame_upload_batch(sdv_ctx* c, int n, const uint64_t* frames, const float* const* imgs_wh, const float* exposures);
/* Uploads are ASYNCHRONOUS on a dedicated ingest stream so that they overlap the tracking of the previous batch: pinned host
 * buffers must stay valid until the next call that synchronises (sdv_sync, any tracker/BA call, sdv_frame_download).
 * _u8: level-0 input in the sensor wire format (sensor_msgs/Image mono8, what src/main.cpp:537-560 receives) — the
 * u8->float conversion of the ingest (DatasetReader.h:152-155, Undistort crop without photometric calibration) is fused
 * into the level-0 kernel; 4x less PCIe traffic.   _dev: level-0 images already in device memory (kernel-only timing). */
int  sdv_frame_upload_batch_u8(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* imgs_wh, const float* exposures);
/* RAW ingest — Undistort::undistort<unsigned char> (util/Undistort.cpp:341-435) + PhotometricUndistorter::processFrame (:177-214), what
 * src/main.cpp:537-560 runs on every sensor_msgs/Image before FullSystem::addActiveFrame.  sdv_set_undistort hands over, once per calibration,
 * the tables the reference's Undistort object holds after readFromFile (:842-886): remapX/remapY (w*h floats of the RECTIFIED size given to
 * sdv_create, source coordinates in the raw w_org x h_org image, -1 = outside), the scalar `factor` of the uncalibrated path, and optionally the
 * inverse response G[256] and the inverse vignette (w_org*h_org) of the photometric calibration (both NULL for KITTI: no pcalib).  A response is
 * applied to frames uploaded with exposure > 0 only (:185).  _raw_u8 then takes native-size mono8 images; rectification, photometric stage and the
 * level-0/level-1 pyramid build are ONE kernel.  Entries that would read outside the raw image are refused (SDV_ERR_ARG). */
int  sdv_set_undistort(sdv_ctx* c, int w_org, int h_org, const float* remapX, const float* remapY, float factor, const float* G256, const float* vignette_inv);
int  sdv_frame_upload_batch_raw_u8(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* raw_imgs_worg_horg, const float* exposures);
/* RAW ingest of several cameras in one context: one Undistort object per calibration file (util/Undistort.cpp:232-334, what src/main.cpp builds once
 * per sequence), kept side by side.  sdv_set_undistort_cam sets or replaces camera `cam`'s tables, with the arguments and checks of sdv_set_undistort;
 * the raw size w_org x h_org is per camera, the remap tables have the camera's rectified size (sdv_set_camera_size; the context's w*h unless set).  Replacing a camera is stream-ordered: an
 * ingest already enqueued finishes with the old tables; the other cameras are untouched.  sdv_set_undistort is this call with cam = 0.
 * sdv_frame_upload_batch_raw_u8_cams: image k is native w_org x h_org mono8 of camera cams[k], rectified with that camera's tables in the same one
 * kernel (cams == NULL: every image is camera 0, which is sdv_frame_upload_batch_raw_u8), into a frame of that camera's rectified size.  Example: the
 * KITTI odometry calibrations (calib/KITTI/00.txt, 03.txt, 04.txt) come in three raw sizes, 1241x376, 1242x375 and 1226x370, that all crop to 1200x360
 * with different rectified K: one camera each, every sequence's tracker slots bound to its camera's K with sdv_set_calib_slots, and all sequences
 * ingested in one batch.  cams is checked before anything else: an index outside [0, SDV_MAX_CAMERAS) returns SDV_ERR_ARG, a camera that was never set
 * SDV_ERR_STATE, and a refused call changes no frame. */
#define SDV_MAX_CAMERAS 8
int  sdv_set_undistort_cam(sdv_ctx* c, int cam, int w_org, int h_org, const float* remapX, const float* remapY, float factor, const float* G256, const float* vignette_inv);
int  sdv_frame_upload_batch_raw_u8_cams(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* raw_imgs, const int32_t* cams, const float* exposures);
/* FullSystem::setGammaFunction (FullSystem.cpp:225-249) for camera `cam`: BInv256 is the array the reference passes, PhotometricUndistorter::getG()
 * (src/main.cpp sets it from the same calibration as the camera's Undistort).  Its inverse B weighs every absSquaredGrad the frames of this camera get:
 * |grad|^2 * gw^2 with gw = B[c+1]-B[c], c = (int)(I+0.5f) clamped to [5, 250] (FrameHessian::makeImages, HessianBlocks.cpp:158-164, with the default
 * setting_gammaWeightsPixelSelect = 1).  That is what the PixelSelector reads (makeHists level 0, makeMaps / makeMapsFromLidar levels 0..2: makeNewTraces
 * and the LiDAR initialiser) and what sdv_frame_download returns as abs_out; the gradients themselves and every tracker / back-end input are unweighted.
 * BInv256 == NULL restores the identity B[i] = i (gw = 1), which a camera has until this is called.  The reference sets the gamma before its first frame:
 * SDV_ERR_STATE while a frame of this camera is resident; SDV_ERR_ARG for a camera outside [0, SDV_MAX_CAMERAS).  A refused call changes nothing. */
int  sdv_set_gamma_cam(sdv_ctx* c, int cam, const float* BInv256);
int  sdv_frame_build_batch_dev(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs_dev, int fmt, const float* exposures);
/* fmt: 0 float (copied into frame storage), 1 mono8, 2 float ADOPTED as the frame's level-0 plane (zero copy: the buffer must stay
 * valid and unmodified until sdv_frame_release / the handle is re-uploaded — for producers that already write into device memory). */
/* Cameras of different rectified sizes in one context (KITTI 1200x360 next to KITTI-360 1400x360).  Camera 0 always has the context size (sdv_create's
 * w, h); cameras 1..SDV_MAX_CAMERAS-1 start at it.  sdv_set_camera_size gives camera `cam` another rectified size w x h: w <= the context's w, h <= its
 * h (the reprojection grid, tracker-slot clouds and keyframe-rate scratch have the context size: create the context at the largest size), and the
 * context's pyramid depth valid at that size (even w, h when levels > 1, every level non-empty).  Frames are stored in the context's pool at the context
 * size unless the camera has a pool of its own at its size (sdv_set_camera_storage).  Camera 0, a camera index out of range or a size outside these rules
 * return SDV_ERR_ARG; resizing a camera that has Undistort tables, a resident frame, a bound tracker or selector slot (sdv_set_calib_slots_cams,
 * sdv_selector_set_slot_cams) or a frame pool of its own returns SDV_ERR_STATE.  A refused call changes nothing.
 * sdv_set_undistort_cam then takes remap tables of that camera's size.  A frame has the size of the camera it was ingested for:
 * sdv_frame_upload_batch_cams takes host float (fmt 0) or mono8 (fmt 1) images, and sdv_frame_build_batch_dev_cams device images with the fmt values of
 * sdv_frame_build_batch_dev (fmt 2 adopts a buffer of w_cam*h_cam floats), each at its camera's size.  cams == NULL is camera 0 (the entries without
 * _cams); every camera index is checked before any frame is claimed or anything is enqueued.
 * Every per-frame entry compares the frame's size with its slot's and returns SDV_ERR_ARG on a mismatch, changing no state: sdv_tracker_set_ref (ref
 * frame), calc_res / track / track_batch / sdv_track_new_coarse_batch (new frame), sdv_map_set (host keyframes), sdv_reproject_map_batch /
 * sdv_tracker_refine_batch (target frame); sdv_ba_set_window needs all frames of one window at one size.  The keyframe-rate candidate management
 * (selector, makeNewTraces, activation, immature points, LiDAR front-end) names a camera per job (the _cam / _cams entries, sdv_selector_set_slot_cams)
 * and works at that camera's size; a frame of another size returns SDV_ERR_ARG and changes no state.  The entries without _cam(s) are camera 0. */
int  sdv_set_camera_size(sdv_ctx* c, int cam, int w, int h);
/* Frame storage per camera.  sdv_create allocates the context pool: max_frames frames and max_kf_images keyframe level-0 images at the context size, for
 * every camera.  sdv_set_camera_storage gives camera `cam` (1..SDV_MAX_CAMERAS-1) a pool of its own at its rectified size (sdv_set_camera_size):
 * max_frames frames and max_kf_images keyframe level-0 images (0: the default of sdv_settings::max_kf_images; at most max_frames).  The storage depth stays
 * the context's `levels`.  From then on every frame of the camera is claimed from that pool and its keyframe images too, with no fallback to the context
 * pool: a full pool returns SDV_ERR_CAPACITY.  A handle resident in another pool than its new camera's moves when it is uploaded again: every image of
 * the upload is given its frame first, and a full pool (SDV_ERR_CAPACITY) or a pinned handle (SDV_ERR_STATE) refuses the whole upload with every handle
 * left as it was; then each moved handle's old frame is released as sdv_frame_release would.  Adopted level-0 buffers (fmt 2) work as before: only the levels >= 1 and the texel caches come from the pool.  max_frames == 0 drops the
 * camera's pool: its frames come from the context pool again.  Camera 0, a camera out of range or a negative count return SDV_ERR_ARG; replacing or
 * dropping a pool while one of its frames is resident or one of its keyframe images is taken returns SDV_ERR_STATE.  All-or-nothing: the new pool is
 * allocated before the old one is freed, and a failed allocation returns SDV_ERR_CUDA with the old pool in place.  Waits for the context's streams.
 * sdv_camera_storage_bytes: the device bytes of one frame and of one keyframe level-0 image of camera `cam` (0..SDV_MAX_CAMERAS-1) as they are stored now
 * (its own pool, or the context size); either pointer may be NULL.  A frame is 4 w h + 20 P bytes with P = sum over levels l >= 1 of (w>>l)(h>>l), a
 * keyframe image 16 w h. */
int  sdv_set_camera_storage(sdv_ctx* c, int cam, int max_frames, int max_kf_images);
int  sdv_camera_storage_bytes(sdv_ctx* c, int cam, uint64_t* frame_bytes, uint64_t* kf_image_bytes);
/* Cameras of different pyramid depths in one context (pyrLevelsUsed, util/globalCalib.cpp:22-30: KITTI-CARLA's 1392x1024 has 5 levels, KITTI's 1200x360 4).
 * sdv_create's `levels` is the STORAGE depth: every frame is built to it, whatever its camera.  A camera's depth is what its tracker / map slots and jobs
 * use, as the reference's pyrLevelsUsed: sdv_tracker_set_ref builds clouds for that many levels, trackNewestCoarse starts at depth - 1 by default
 * (sdv_tracker_track_batch_levels, sdv_track_new_coarse_batch: FullSystem.cpp:421), and the Reprojector's search level is capped at depth - 1
 * (Reprojector.cpp:268; sdv_reproject_map_batch, sdv_tracker_refine_batch).  sdv_tracker_set_cloud / _get_cloud / _calc_res refuse a level at or past the
 * slot camera's depth, sdv_frame_download one at or past the frame camera's depth (SDV_ERR_ARG).  BA and immature points read level 0, the activation
 * walk and distance map level 1, the selector levels 0..2: they do not depend on the depth.
 * sdv_set_camera_levels gives camera `cam` (camera 0 included) the depth `levels` in 1..the context's `levels`; every camera starts at the context's
 * depth.  The reference rule is levels = sdv_pyr_levels(w_cam, h_cam).  A size valid for sdv_set_camera_size is valid at every smaller depth.  A camera
 * or depth out of range returns SDV_ERR_ARG; SDV_ERR_STATE while a tracker slot bound to the camera holds a reference or a resident map (built at the old
 * depth), or for a depth below 3 while a selector slot is bound to the camera (sdv_selector_set_slot_cams refuses such a camera with SDV_ERR_ARG).
 * A refused call changes nothing.  sdv_set_calib_slots_cams refuses to move a slot holding a reference or map to a camera of another size OR depth. */
int  sdv_set_camera_levels(sdv_ctx* c, int cam, int levels);
int  sdv_frame_upload_batch_cams(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs, const int32_t* cams, int fmt, const float* exposures);
int  sdv_frame_build_batch_dev_cams(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs_dev, const int32_t* cams, int fmt, const float* exposures);
int  sdv_frame_release(sdv_ctx* c, uint64_t frame);
/* test hook: copy one level back as AoS {I,dx,dy} (w*h*3 floats) and absSquaredGrad (w*h floats); either may be NULL */
int  sdv_frame_download(sdv_ctx* c, uint64_t frame, int lvl, float* dI3_out, float* abs_out);

/* ---- tracker reference: CoarseTracker::makeK :77-106 is sdv_create / sdv_set_calib (context) and sdv_set_calib_slots (per instance) -----------
 * CoarseTracker::setCoarseTrackingRef / setCTRefForFirstFrame  CoarseTracker.cpp:636-660 -> makeCoarseDepthL0 :258-425.
 * The PointHessian graph walk (:264-294) stays on the host: the caller passes one row per splat, {u,v,idepth,HdiF},
 * with round_half[i]=0 for `int(u)` (newest-KF sensor points, :270-271) or 1 for `int(u+0.5f)` (:116-117, :285-286). */
int  sdv_tracker_set_ref(sdv_ctx* c, int slot, uint64_t ref_frame, int n, const float* pts4, const int32_t* round_half,
                         float ref_exposure_unused, double ref_a, double ref_b);
/* setCoarseTrackingRef for n tracker slots in one launch sequence (makeKeyFrame of many sequences).  Job j is sdv_tracker_set_ref(slots[j], ref_frames[j],
 * rows pt_begin[j] .. pt_begin[j+1] of pts4 / round_half, ref_ab[2j], ref_ab[2j+1]) at its slot camera's size and depth; ref_ab == NULL is (0, 0) for every
 * job.  Two jobs may share a reference frame.  npts_out[j*SDV_PYR_LEVELS + l] (may be NULL) = job j's true cloud size at level l, 0 past its camera's depth.
 * The clouds are bit-identical to n single calls; sdv_tracker_set_ref is this call with n = 1.  n == 0 returns SDV_OK.
 * Refused before anything is enqueued, changing no slot: a NULL array, pt_begin[0] != 0 or decreasing, a slot out of range or named twice (SDV_ERR_ARG);
 * an unknown frame (SDV_ERR_NOFRAME); a frame of another size than its slot's camera, or a splat outside its slot camera's image (SDV_ERR_ARG).
 * Over capacity (max_ref_points): every job whose clouds fit is installed; every job with a level over its slot's capacity is left with NO reference (as
 * sdv_tracker_set_ref leaves its slot), and the call returns SDV_ERR_CAPACITY naming the first such job, with npts_out filled.
 * Launches: a fixed number per chunk of jobs whose planes fit the build's plane budget (DESIGN.md Round 13), whatever the splat count or multiplicity;
 * one host wait per call.  Counted by sdv_launch_count, timed by sdv_last_kernel_ms. */
int  sdv_tracker_set_ref_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* ref_frames, const int32_t* pt_begin, const float* pts4,
                               const int32_t* round_half, const double* ref_ab, int32_t* npts_out);
/* direct injection / readback of one level's reference cloud pc_u,pc_v,pc_idepth,pc_color (tests, stress config) */
int  sdv_tracker_set_cloud(sdv_ctx* c, int slot, uint64_t ref_frame, int lvl, int n, const float* u, const float* v,
                           const float* idepth, const float* color, double ref_a, double ref_b);
int  sdv_tracker_get_cloud(sdv_ctx* c, int slot, int lvl, int* n, float* u, float* v, float* idepth, float* color);

/* ---- tracker residual + Gauss-Newton system (one fused kernel launch) ---------------------------------------------
 * Vec6 CoarseTracker::calcRes(int lvl, const SE3& refToNew, AffLight aff_g2l, float cutoffTH)   CoarseTracker.cpp:486-634
 * void CoarseTracker::calcGSSSE(int lvl, Mat88& H_out, Vec8& b_out, const SE3&, AffLight)        CoarseTracker.cpp:427-484
 * calc_res evaluates residuals AND accumulates the 9x9 system of the same pose in one pass; calc_gs returns the
 * (scaled, /n) H,b of the last calc_res on that slot, exactly the state calcGSSSE would read from buf_warped_*. */
int  sdv_tracker_calc_res(sdv_ctx* c, int slot, uint64_t new_frame, int lvl, const double T[7], double a, double b,
                          float cutoffTH, double rs_out[6]);
int  sdv_tracker_calc_gs(sdv_ctx* c, int slot, int lvl, double H88_out[64], double b8_out[8]);

/* ---- device-resident coarse-to-fine LM ------------------------------------------------------------------------------
 * bool CoarseTracker::trackNewestCoarse(FrameHessian*, SE3& lastToNew_out, AffLight& aff_g2l_out, int coarsestLvl,
 *                                       Vec5 minResForAbort, Output3DWrapper*)                  CoarseTracker.cpp:662-838
 * T_io/ab_io are in-out like lastToNew_out/aff_g2l_out (written only when the call is not aborted, as in the reference);
 * lastRes = CoarseTracker::lastResiduals, flow = lastFlowIndicators (CoarseTracker.h:57-65). */
typedef struct {
  int64_t point_evals[SDV_PYR_LEVELS];   /* sum of pc_n[lvl] over all calcRes evaluations (roofline accounting) */
  int32_t iterations[SDV_PYR_LEVELS];
  int32_t accepts[SDV_PYR_LEVELS];
} sdv_track_stats;
int  sdv_tracker_track(sdv_ctx* c, int slot, uint64_t new_frame, double T_io[7], double ab_io[2], int coarsest,
                       const double minResForAbort[5], double lastRes[5], double flow[3], int* good, sdv_track_stats* stats);
/* batched mode (north_star: independent sequences / Monte-Carlo re-runs): n independent trackNewestCoarse calls in ONE
 * launch, one thread-block cluster each.  Arrays are n x the single-call shapes. */
int  sdv_tracker_track_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* new_frames, double* T_io, double* ab_io,
                             int coarsest, const double* minResForAbort, double* lastRes, double* flow, int32_t* good,
                             sdv_track_stats* stats);
/* the same with a coarsest level per job: job k starts at coarsest[k]; coarsest == NULL starts every job at its slot camera's depth - 1 (pyrLevelsUsed-1,
 * sdv_set_camera_levels).  sdv_tracker_track_batch is this call with its scalar for every job.  A level at or past a job's depth, or >= 5
 * (CoarseTracker.cpp:672), returns SDV_ERR_ARG before anything is enqueued. */
int  sdv_tracker_track_batch_levels(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* new_frames, double* T_io, double* ab_io,
                                    const int32_t* coarsest, const double* minResForAbort, double* lastRes, double* flow, int32_t* good,
                                    sdv_track_stats* stats);
/* ---- map reprojection + direct feature alignment (SURVEY.md §8 a10): the Reprojector of FullSystem::trackNewCoarse / makeKeyFrame
 *   void Reprojector::reprojectMap(FrameHessian* frame, std::vector<std::pair<PointHessian*, Eigen::Vector2d>>& overlap_pts)     Reprojector.cpp:117-156
 *   void Reprojector::backprojectMap(FrameHessian* ref_frame, FrameHessian* frame, overlap_pts&)                                   :158-185
 *   with reprojectPoint :600-616, reprojectCell :198-233, findMatchDirect :235-292, getWarpMatrixAffine :14-37, getBestSearchLevel :39-51,
 *   warpAffine :53-86, align1D :346-455, align2D :457-560 (options_: find_match_direct = true, align_max_iter = 10; grid cell 25 px).
 * sdv_map_set     makes the active map of one sequence resident (per keyframe): the window's keyframes (frameHessians_ order: device frame
 *                 handle, shell->camToWorld, shell->aff_g2l {a,b}) and their ACTIVE PointHessians grouped by host in that order
 *                 (u, v, idepth, host index, type 0 CORNER / 1 EDGELET).  `slot` shares the index space of the tracker slots.
 * sdv_reproject_map_batch   n independent reprojectMap calls in one launch sequence.  Per job: map slot, target frame handle + camToWorld +
 *                 aff_g2l, cur_kf_index (index of the target in the map's keyframes or -1), only_host (-1: reprojectMap over all keyframes in
 *                 close_kfs order; h: backprojectMap of keyframe h's points), backup (Reprojector::backup, selects the reference keyframe when
 *                 there are <= 2 keyframes, :242-250).  cell_order[n_cols*n_rows] is the grid visiting order (the reference shuffles it with
 *                 rand(), :111; NULL = identity); max_matches = (int)(0.8*setting_desiredImmatureDensity).
 *                 Outputs per job k, in visiting order: n_out[k] matches, out_pt[k*cells + i] = index into the slot's points,
 *                 out_px[(k*cells + i)*2] = aligned pixel (it->px).
 *                 Cameras of a smaller size (sdv_set_camera_size): n_cols x n_rows and cells are the CONTEXT grid (sdv_reproject_grid), and so is
 *                 cell_order.  A job whose slot's camera is w x h has the grid ceil(w/25) x ceil(h/25), numbered row-major in its own columns; it walks
 *                 cell_order and skips every context cell (col, row) = (cell % n_cols, cell / n_cols) with col >= ceil(w/25) or row >= ceil(h/25), and
 *                 visits the others as its cell row*ceil(w/25) + col.  That subsequence is a permutation of the job's grid, so one context order
 *                 serves a mixed batch, and the job gets the matches a context of its own size gives for the filtered order.  The output stride
 *                 stays the context's cells.  sdv_tracker_refine_batch and sdv_track_new_coarse_batch apply the same rule. */
typedef struct { float u, v, idepth; int32_t host; int32_t type; } sdv_map_pt;
int  sdv_reproject_grid(sdv_ctx* c, int* n_cols, int* n_rows);
int  sdv_map_set(sdv_ctx* c, int slot, int nH, const uint64_t* host_frames, const double* host_T7, const double* host_ab, int nP, const sdv_map_pt* pts);
/* sdv_map_set for n slots: job j has the keyframes host_begin[j] .. host_begin[j+1] of host_frames / host_T7 / host_ab (may be NULL: every ab = (0, 0)) and
 * the points pt_begin[j] .. pt_begin[j+1] of pts, whose `host` field indexes the job's own keyframes.  All-or-nothing: every check of sdv_map_set runs for
 * every job, and a slot named twice or host_begin[0] / pt_begin[0] != 0 returns SDV_ERR_ARG, before any slot, pin or buffer changes.  Pins follow
 * sdv_map_set.  The call waits for the device twice whatever n is: before it overwrites slots an earlier launch may read, and after its one upload. */
int  sdv_map_set_batch(sdv_ctx* c, int n, const int32_t* slots, const int32_t* host_begin, const uint64_t* host_frames, const double* host_T7,
                       const double* host_ab, const int32_t* pt_begin, const sdv_map_pt* pts);
/* A resident map slot (and a resident BA window, below) REFERENCES the device images of its keyframes: while it does, sdv_frame_release /
 * re-uploading one of those handles returns SDV_ERR_STATE instead of handing the storage to another frame under the reader.  sdv_map_set on
 * the same slot replaces the references; sdv_map_clear drops them (the FrameHessian destructor path of a marginalised keyframe). */
int  sdv_map_clear(sdv_ctx* c, int slot);
int  sdv_reproject_map_batch(sdv_ctx* c, int n_jobs, const int32_t* slots, const uint64_t* cur_frames, const double* cur_T7, const double* cur_ab,
                             const int32_t* cur_kf_index, const int32_t* only_host, const int32_t* backup, const int32_t* cell_order, int max_matches,
                             int32_t* n_out, int32_t* out_pt, double* out_px);

/* ---- semi-direct pose refinement on matched map points (SURVEY.md §8 a11)
 * bool CoarseTracker::structPoseEstimation(SE3& curToWorld, std::vector<std::pair<PointHessian*, Eigen::Vector2d>>& overlap_pts)
 *                                                                                              CoarseTracker.cpp:949-1007
 *   with calculateRes :840-871, calculateWeight :873-887, calcHandb :889-947 (called from FullSystem::trackNewCoarse, FullSystem.cpp:483-488).
 * One overlap point = the PointHessian fields the function reads (u, v, idepth, host) + the matched pixel (it->second cast to float).
 * `host` indexes the job's host_T7 rows = host->shell->camToWorld of the distinct host keyframes.  curToWorld_io is in-out like the
 * reference argument (written only by accepted steps).  res = final mean squared reprojection error (resOld), iterations/accepts = loop
 * statistics.  Batched: job k owns pts[pt_begin[k] .. pt_begin[k+1]) and host_T7 rows [host_begin[k] .. host_begin[k+1]) (<= 16 hosts). */
typedef struct { float u, v, idepth; int32_t host; float obs_x, obs_y; } sdv_overlap_pt;
int  sdv_tracker_struct_pose(sdv_ctx* c, int n, const sdv_overlap_pt* pts, int nH, const double* host_T7, double curToWorld_io[7],
                             float* res, int* iterations, int* accepts);
int  sdv_tracker_struct_pose_batch(sdv_ctx* c, int n_jobs, const int32_t* pt_begin, const sdv_overlap_pt* pts, const int32_t* host_begin,
                                   const double* host_T7, double* curToWorld_io, float* res, int32_t* iterations, int32_t* accepts);
/* the same with the K of the tracker slot each job belongs to (structPoseEstimation is a CoarseTracker member, CoarseTracker.cpp:949-1007);
 * slots == NULL is sdv_tracker_struct_pose_batch (every job on the context calibration). */
int  sdv_tracker_struct_pose_batch_slots(sdv_ctx* c, int n_jobs, const int32_t* slots, const int32_t* pt_begin, const sdv_overlap_pt* pts, const int32_t* host_begin,
                                         const double* host_T7, double* curToWorld_io, float* res, int32_t* iterations, int32_t* accepts);
/* ---- fused per-frame refinement (the tail of FullSystem::trackNewCoarse, FullSystem.cpp:482-488): reprojectMap(fh) -> structPoseEstimation
 * without leaving the device.  curToWorld_io: fh->shell->camToWorld from the photometric tracker in, refined pose out; cur_ab = the tracked
 * aff_g2l.  n_matches = overlap_pts.size(), res/iterations/accepts as in sdv_tracker_struct_pose_batch. */
int  sdv_tracker_refine_batch(sdv_ctx* c, int n_jobs, const int32_t* slots, const uint64_t* cur_frames, double* curToWorld_io, const double* cur_ab,
                              const int32_t* cell_order, int max_matches, int32_t* n_matches, float* res, int32_t* iterations, int32_t* accepts);
/* ---- Vec4 FullSystem::trackNewCoarse(FrameHessian* fh)                                                   FullSystem.cpp:283-500 (§8 a4)
 * The per-frame policy for a running system (allFrameHistory.size() > 2): 31 motion hypotheses (:334-395), the re-track loop over
 * trackNewestCoarse with the achievedRes abort vector (:410-462), fallback (:464-470), pose composition (:474-479), reprojectMap +
 * structPoseEstimation (:481-488).  Batched over n sequences: try i is one track_batch launch over the sequences still searching.
 * The caller keeps FullSystem's per-sequence state (allFrameHistory shells, lastCoarseRMSE, firstCoarseRMSE) and passes what the function reads. */
typedef struct {
  /* in */
  int32_t  slot;                 /* tracker slot == map slot of the sequence (coarseTracker / the active window) */
  int32_t  poses_valid;          /* 1: slast->poseValid && sprelast->poseValid && lastF->shell->poseValid (:390) -> 31 hypotheses; 0: -> identity only (:391-394);
                                    2: the second frame of a sequence (allFrameHistory.size() == 2, :299-331) -> identity + 52 pure rotations, no history needed */
  uint64_t frame;                /* device handle of fh */
  double   sprelast_c2w[7], slast_c2w[7], lastF_c2w[7];   /* camToWorld of allFrameHistory[size-3], [size-2], coarseTracker->lastRef->shell */
  double   aff_last[2];          /* slast->aff_g2l {a,b} */
  /* in-out */
  double   lastCoarseRMSE[5];    /* FullSystem::lastCoarseRMSE in, achievedRes out (:472) */
  /* out */
  double   camToWorld[7];        /* fh->shell->camToWorld after structPoseEstimation */
  double   camToTrackingRef[7];  /* fh->shell->camToTrackingRef (:490-491) */
  double   aff_g2l[2];           /* fh->shell->aff_g2l */
  double   flow[3];              /* flowVecs (the Vec4 result is {lastCoarseRMSE[0], flow[0..2]}) */
  float    refine_res;
  int32_t  have_one_good, tries, n_matches, refine_iterations, refine_accepts;
} sdv_track_new_coarse_io;
int  sdv_track_new_coarse_batch(sdv_ctx* c, int n, sdv_track_new_coarse_io* io, const int32_t* cell_order, int max_matches);
/* lastF_2_fh_tries[i] of FullSystem.cpp:346-394 for one job (host arithmetic only, no device needed); n_tries = 31, or 1 when the pose history is invalid */
int  sdv_track_hypothesis(const sdv_track_new_coarse_io* io, int i, double T7_out[7], int* n_tries);

/* device time of the last track / track_batch / calc_res launch in milliseconds (CUDA events on the context stream) */
float sdv_last_kernel_ms(sdv_ctx* c);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
long long sdv_launch_count(sdv_ctx* c);
/* bytes copied H2D and again D2H per trackNewestCoarse job (the job descriptor carries inputs and results) */
int  sdv_track_job_bytes(void);


/* ---- immature points (SURVEY.md §8f rank 2): candidate construction and epipolar tracing
 *   ImmaturePoint::ImmaturePoint(int u, int v, FrameHessian* host, float type, CalibHessian*)               FullSystem/ImmaturePoint.cpp:8-36
 *   ImmaturePointStatus ImmaturePoint::traceOn(FrameHessian* frame, const Mat33f& hostToFrame_KRKi, const Vec3f& hostToFrame_Kt,
 *                                              const Vec2f& hostToFrame_affine, CalibHessian*, bool)           FullSystem/ImmaturePoint.cpp:50-352
 *   called for every immature point of every active keyframe by FullSystem::traceNewCoarse                     FullSystem/FullSystem.cpp:519-552
 * The record mirrors the members of ImmaturePoint the two functions read or write (ImmaturePoint.h:33-78); it stays with the caller (the reference keeps the
 * points in host->immaturePoints), the device works on a copy per call.  lastTraceStatus: 0 GOOD, 1 OOB, 2 OUTLIER, 3 SKIPPED, 4 BADCONDITION, 5 UNINITIALIZED. */
typedef struct {
  float u, v, idepth_min, idepth_max;
  float color[8], weights[8], gradH[4];           /* gradH: Mat22f row-major */
  float energyTH, quality, lastTraceUV[2], lastTracePixelInterval;
  int32_t lastTraceStatus;
} sdv_immature_pt;
/* constructor for n candidates at integer pixels uv[2n] of a resident keyframe (>= 3 px from the border, else SDV_ERR_ARG).  _cam: the keyframe is camera cam's
 * (its size must be that camera's, and the border is that camera's); sdv_immature_init is camera 0. */
int  sdv_immature_init(sdv_ctx* c, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out);
int  sdv_immature_init_cam(sdv_ctx* c, int cam, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out);
/* traceOn for n_groups (host keyframe, traced frame) pairs in ONE launch: group g traces pts_io[pt_begin[g] .. pt_begin[g+1]) against frames[g] with
 * KRKi9[9g..] = K R K^-1 (row-major), Kt3[3g..] = K t of hostToNew and aff2[2g..] = AffLight::fromToVecExposure(host, new) — what traceNewCoarse computes per host
 * (:532-538).  Groups may belong to different sequences (batched mode).  pts_io is updated in place; status_out (n points) may be NULL.
 * _cams: group g traces at camera cams[g]'s size (wG[0], hG[0] of its sequence) and frames[g] must have that size; cams == NULL is sdv_immature_trace_batch (camera 0). */
int  sdv_immature_trace_batch(sdv_ctx* c, int n_groups, const uint64_t* frames, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* aff2,
                              sdv_immature_pt* pts_io, int32_t* status_out);
int  sdv_immature_trace_batch_cams(sdv_ctx* c, int n_groups, const uint64_t* frames, const int32_t* cams, const int32_t* pt_begin, const float* KRKi9, const float* Kt3,
                                   const float* aff2, sdv_immature_pt* pts_io, int32_t* status_out);
/* Activation — PointHessian* FullSystem::optimizeImmaturePoint(ImmaturePoint*, int minObs, ImmaturePointTemporaryResidual*)   FullSystemOptPoint.cpp:18-183
 * over ImmaturePoint::linearizeResidual (ImmaturePoint.cpp:410-476): Gauss-Newton on the inverse depth of a candidate against every other keyframe of the window.
 * Group g = the candidates pts[pt_begin[g] .. pt_begin[g+1]) of ONE host keyframe; its targets are entries tgt_begin[g] .. tgt_begin[g+1]) of target_frames / pre14
 * (frameHessians without the host, window order; pre14 = host->targetPrecalc[target]: PRE_RTll[9] row-major, PRE_tTll[3], PRE_aff_mode[2]); calib6[6g..] = fxl fyl cxl cyl
 * fxli fyli of the CalibHessian.  Outputs per candidate: status 0 = not well constrained (stays immature; the function's `return 0`), -1 = outlier / non-finite
 * (deleted), 1 = activated with idepth_out (setIdepth/setIdepthZero) and res_state_out[k*res_stride + i] = final state of the temporary residual to target i
 * (0 IN -> a PointFrameResidual is created, 1 OOB, 2 OUTLIER; -1 = unused).  The PointHessian / PointFrameResidual objects stay with the caller.
 * _cams: group g works at camera cams[g]'s size and every target of the group must have it; cams == NULL is sdv_immature_optimize_batch (camera 0). */
int  sdv_immature_optimize_batch(sdv_ctx* c, int n_groups, const int32_t* pt_begin, const int32_t* tgt_begin, const uint64_t* target_frames, const float* pre14, const float* calib6,
                                 int min_obs, const sdv_immature_pt* pts, const uint8_t* is_from_sensor, int res_stride, int32_t* status_out, float* idepth_out, int32_t* res_state_out);
int  sdv_immature_optimize_batch_cams(sdv_ctx* c, int n_groups, const int32_t* pt_begin, const int32_t* tgt_begin, const uint64_t* target_frames, const float* pre14,
                                      const float* calib6, const int32_t* cams, int min_obs, const sdv_immature_pt* pts, const uint8_t* is_from_sensor, int res_stride,
                                      int32_t* status_out, float* idepth_out, int32_t* res_state_out);
/* ---- device-resident immature points: FrameHessian::immaturePoints (HessianBlocks.h) kept on the device, one block per host keyframe, keyed by its frame handle.
 * The records are made on the device (makeNewTraces), traced there every frame (traceNewCoarse) and never need to visit the host; the entries above copy every
 * record to the device and back per call.  A block holds, per point, the sdv_immature_pt record and the sdv_immature_meta record below, in the order of
 * host->immaturePoints.  Tracker call domain.  The pool grows at keyframe rate only (set, make_new_traces_store); the per-frame trace never allocates.
 * A host with no block returns SDV_ERR_NOFRAME from every entry that names it; a refused call changes no block.
 * sdv_immature_store_set    replaces host_frame's block by pts[n] (+ meta[n]; NULL: my_type 1, type -1, not from the sensor); n == 0 leaves an empty block.
 *                           The frame need not be resident: the records carry all the trace reads of their host.
 * sdv_immature_store_count  counts_out[i] = size of hosts[i]'s block, for n hosts.
 * sdv_immature_store_get    reads host_frame's block back in its current order; *n_out = its size (also when SDV_ERR_CAPACITY: cap < size, nothing copied);
 *                           pts_out / meta_out may each be NULL.
 * sdv_immature_store_drop   drops the blocks of n hosts: the keyframe leaves the window (FullSystem::marginalizeFrame -> FrameHessian::release deletes its immaturePoints,
 *                           HessianBlocks.cpp:90-105). */
typedef struct { float my_type; int32_t type; int32_t isFromSensor; float idepth_fromSensor; } sdv_immature_meta;   /* ImmaturePoint members of the activation / PointHessian ctor */
int  sdv_immature_store_set(sdv_ctx* c, uint64_t host_frame, int n, const sdv_immature_pt* pts, const sdv_immature_meta* meta);
int  sdv_immature_store_count(sdv_ctx* c, int n, const uint64_t* hosts, int32_t* counts_out);
int  sdv_immature_store_get(sdv_ctx* c, uint64_t host_frame, int cap, sdv_immature_pt* pts_out, sdv_immature_meta* meta_out, int32_t* n_out);
int  sdv_immature_store_drop(sdv_ctx* c, int n, const uint64_t* hosts);
/* FullSystem::traceNewCoarse (FullSystem.cpp:519-552) on the store: group g traces every point of hosts[g]'s block into frames[g] (camera cams[g]'s size; NULL: camera 0)
 * with KRKi9[9g..], Kt3[3g..], aff2[2g..] as sdv_immature_trace_batch_cams takes them (:534-538); ImmaturePoint::traceOn (ImmaturePoint.cpp:50-352) updates the records in
 * place.  Groups of several sequences and cameras go into one launch; a host may appear in one group per call (else SDV_ERR_ARG).  counts_out (may be NULL):
 * counts_out[6g + s] = the points of group g whose lastTraceStatus is s afterwards (0 GOOD .. 5 UNINITIALIZED: trace_good, trace_oob, ... of :543-548).
 * No record crosses PCIe; the call returns without waiting for the device unless counts_out is given.  Until that kernel has run, re-ingesting a traced frame
 * (or a frame into its storage after sdv_frame_release) is ordered after it on the device, and releasing an adopted frame waits for it on the host. */
/* void FullSystem::activatePointsMT() (FullSystem.cpp:598-720) on the store, after the currentMinActDist update (:571-592, which reads ef->nPoints and stays with the caller),
 * for n sequences.  Sequence j's window is hosts[host_begin[j] .. host_begin[j+1]) in frameHessians order, newest last (1..16 keyframes, at most SDV_MAX_FRAMES_WINDOW
 * targets each); per window host: flagged[] = flaggedForMarginalization, cKRKi9 / cKt3 = K[1] R K[0]^-1, K[1] t of host -> newest (:606-610).  The ACTIVE-point sources
 * of the distance map (src_host_begin per sequence, src_pt_begin, KRKi9, Kt3, uvid) and min_act_dist[j] as sdv_activate_select_batch_cams takes them; pre14 = the
 * (host, target) rows of sdv_immature_optimize_batch, host-major over each window, targets in window order without the host; calib6[6j..]; cams[j] (NULL: camera 0).
 * On the device: the deletion / canActivate filter (:612-645, setting_minTraceQuality 3), the distance map and walk (:647-671; a candidate projecting outside level 1 is
 * deleted), optimizeImmaturePoint with minObs 1 on the accepted ones, the post pass (:683-707: activated, -1 and OOB points leave the store) and the swap-with-back
 * compaction of every host's block (:709-720).  Out, in toOptimize order, for the activated points only: act_host (index into hosts), act_idx (idxInImmaturePoints before
 * the compaction), the record and meta, act_idepth, act_res_state[k*SDV_MAX_FRAMES_WINDOW + t] (state of the residual to target t, -1 padding); n_act_out[j] per sequence;
 * counts_out[g] (may be NULL) = host g's block size after the compaction.  More than cap activated points return SDV_ERR_CAPACITY and change nothing. */
int  sdv_activate_points_store_batch(sdv_ctx* c, int n, const int32_t* host_begin, const uint64_t* hosts, const int32_t* flagged, const float* cKRKi9, const float* cKt3,
                                     const int32_t* src_host_begin, const int32_t* src_pt_begin, const float* KRKi9, const float* Kt3, const float* uvid, const float* min_act_dist,
                                     const float* pre14, const float* calib6, const int32_t* cams, int cap, int32_t* n_act_out, int32_t* act_host, int32_t* act_idx,
                                     sdv_immature_pt* act_pts, sdv_immature_meta* act_meta, float* act_idepth, int32_t* act_res_state, int32_t* counts_out);
int  sdv_immature_trace_store_batch(sdv_ctx* c, int n_groups, const uint64_t* hosts, const uint64_t* frames, const int32_t* cams, const float* KRKi9, const float* Kt3,
                                    const float* aff2, int32_t* counts_out);

/* frames + calibration + marginalisation prior:  EnergyFunctional::insertFrame :365-398, setAdjointsF :21-71, HM/bM :88-89.
 * state10 / state_zero10 = FrameHessian::state / state_zero (Vec10: 6 pose, a, b, 2 unused; HessianBlocks.h:141-175),
 * T_evalPT7 = worldToCam_evalPT, calib_value_scaled = CalibHessian::value_scaled {fx,fy,cx,cy}; HM (dim x dim, row-major), bM may be NULL. */
/* =====================================================================================================================
 * Sliding-window back-end: EnergyFunctional + FullSystem::optimize on a FLATTENED window.
 * The reference's pointer graph (FrameHessian -> PointHessian -> PointFrameResidual and the EF* mirrors) stays on the host;
 * the caller passes it in the reference's own iteration order — frames = ef->frames, points = ef->allPoints (contiguous per
 * host frame, EnergyFunctional.cpp:761-782), residuals grouped per point in residualsAll order (res_begin is the CSR row
 * pointer).  This is the makeIDX / insertFrame / insertPoint / insertResidual surface (EnergyFunctional.h:51-72) in one call.
 * ===================================================================================================================== */
int  sdv_ba_set_window(sdv_ctx* c, int nF, const uint64_t* frame_ids, const double* T_evalPT7, const double* state10, const double* state_zero10,
                       const float* ab_exposure, const int32_t* frameID, const float* frameEnergyTH, const double calib_value_scaled[4],
                       const double* HM, const double* bM);
/* CalibHessian::value_zero (HessianBlocks.h:273-289) of a live system: sdv_ba_set_window takes value_zero = value (a fresh CalibHessian); after the first bundle adjustment the two
 * differ and value - value_zero is what the marginalisation prior acts on (EnergyFunctional.cpp:144).  Optional; between sdv_ba_set_window and sdv_ba_set_points.  Units of
 * CalibHessian::value (= value_scaled / SCALE_F resp. SCALE_C).  Oracle side: orc_ba_set_calib_zero, exercised on live windows by tests/test_sequence_ba.py. */
int  sdv_ba_set_calib_zero(sdv_ctx* c, const double value_zero[4]);
/* points + residuals: PointHessian {u,v,idepth,idepth_zero,color[8],weights[8],hasDepthPrior,isFromSensor} (HessianBlocks.h:361-465),
 * PointFrameResidual {host,target,hasMatcher,matcher,isNew} (Residuals.h:30-83).  Runs setPrecalcValues (FullSystem.cpp:1358-1368). */
int  sdv_ba_set_points(sdv_ctx* c, int nP, const float* uv, const float* idepth, const float* idepth_zero, const float* color8, const float* weights8,
                       const int32_t* host, const int32_t* hasDepthPrior, const int32_t* isFromSensor, const int32_t* res_begin,
                       int nR, const int32_t* r_point, const int32_t* r_host, const int32_t* r_target, const int32_t* r_hasMatcher,
                       const float* r_matcher, const int32_t* r_isNew);
/* Vec3 FullSystem::linearizeAll(bool fixLinearization)  FullSystemOptimize.cpp:99-159 -> PointFrameResidual::linearize Residuals.cpp:60-224
 * (+ setNewFrameEnergyTH :63-97; with fix: applyRes + the isNew / toRemove bookkeeping of linearizeAll_Reductor :23-55) */
int  sdv_ba_reset_oob(sdv_ctx* c);                                 /* PointFrameResidual::resetOOB on every residual (optimize :361-362) */
int  sdv_ba_linearize(sdv_ctx* c, int fix, double* energy_out);
int  sdv_ba_apply_res(sdv_ctx* c);                                 /* applyRes_Reductor :57-61 -> Residuals.cpp:252-274, EFResidual::takeDataF */
int  sdv_ba_energy(sdv_ctx* c, double* EL_out, double* EM_out);    /* EnergyFunctional::calcLEnergyF_MT :333-350, calcMEnergyF :284-293 */
/* void EnergyFunctional::solveSystemF(int iteration, double lambda, CalibHessian*)  EnergyFunctional.cpp:650-759
 * (accumulateAF/LF/SCF, stitch, diag-scaled LDLT, orthogonalize for iteration>=2, resubstituteF_MT); x_out[CPARS+6nF] = ef->lastX */
int  sdv_ba_solve(sdv_ctx* c, int iteration, double lambda, double* x_out);
int  sdv_ba_backup(sdv_ctx* c);                                    /* FullSystem::backupState  FullSystemOptimize.cpp:255-300 */
int  sdv_ba_step(sdv_ctx* c, float stepfac, int load_backup, int* canbreak_out);   /* doStepFromBackup :165-250 / loadSateBackup :303-321 */
/* float FullSystem::optimize(int mnumOptIts)  FullSystemOptimize.cpp:344-502 — the whole GN loop incl. the final re-anchoring and
 * linearizeAll(true).  Returns sqrt(lastEnergy / resInA) like the reference. */
int  sdv_ba_optimize(sdv_ctx* c, int mnumOptIts, float* rmse_out, int32_t* iterations_out, int32_t* accepts_out);
float sdv_ba_last_kernel_ms(sdv_ctx* c);                        /* device time of the last sdv_ba_optimize / sdv_ba_optimize_batch (back-end stream) */
/* Batched mode: a context holds any number of independent windows (one per resident sequence).  sdv_ba_select picks the window the
 * set_ / get_ / step-wise calls address (default 0); sdv_ba_optimize_batch runs FullSystem::optimize on n windows at once — every
 * kernel is launched once for all windows and the accept/reject/break decisions are taken on the device. */
int  sdv_ba_select(sdv_ctx* c, int window);
int  sdv_ba_clear(sdv_ctx* c);               /* empty the selected window and drop its references to keyframe images (see sdv_map_clear) */
int  sdv_ba_optimize_batch(sdv_ctx* c, int n, const int32_t* windows, int mnumOptIts, float* rmse_out, int32_t* iterations_out, int32_t* accepts_out);
/* read-back of what the reference leaves in FrameHessian/CalibHessian, PointHessian/EFPoint, PointFrameResidual/EFResidual, EnergyFunctional */
int  sdv_ba_get_frames(sdv_ctx* c, double* T_evalPT7, double* state10, double* step10, float* frameEnergyTH, double* PRE_worldToCam7,
                       double calib_value[4], double calib_step[4]);
int  sdv_ba_get_points(sdv_ctx* c, float* idepth, float* step, float* HdiF, float* bdSumF, float* maxRelBaseline, int32_t* numGoodResiduals, float* idepth_hessian);
/* J24 per residual: {resF[2], Jpdxi[0][6], Jpdxi[1][6], Jpdc[0][4], Jpdc[1][4], Jpdd[2]} = the live part of RawResidualJacobian.h:7-36;
 * energies3 = {state_energy, state_NewEnergy, state_NewEnergyWithOutlier}; states: 0 IN, 1 OOB, 2 OUTLIER (Residuals.h:21) */
int  sdv_ba_get_residuals(sdv_ctx* c, int32_t* state_state, int32_t* state_NewState, float* energies3, int32_t* isActive, float* J24, float* efJ24,
                          float* JpJdF8, float* center3, int32_t* toRemove);
/* ---- keyframe hand-over (SURVEY.md §8 b9): the numeric part of FullSystem::makeKeyFrame after optimize()      FullSystem.cpp:1152-1171
 * sdv_ba_flag_points       FullSystem::flagPointsForRemoval :764-797 for the points the host selected
 *                          (selected[p] = (ph->isOOB(..) || host->flaggedForMarginalization) && ph->isInlierNew(), graph bookkeeping):
 *                          resetOOB + linearize + applyRes(true) + EFResidual::fixLinearizationF (EnergyFunctionalStructs.cpp:46-55) per residual;
 *                          status[p] = 0 untouched / 1 PS_DROP / 2 PS_MARGINALIZE (idepth_hessian > setting_minIdepthH_marg).
 * sdv_ba_marginalize_points EnergyFunctional::marginalizePointsF, EnergyFunctional.cpp:514-576 (addPoint<2>, addPoint(p,false), stitchDouble,
 *                          HM += margWeightFac*(M-Msc)); status==NULL uses the device-resident result of sdv_ba_flag_points.  The accumulation
 *                          order is the order of the status==2 points in the flattened list (= allPointsToMarg when flattened after dropPointsF).
 *                          M, Mb, Msc, Mbsc can be read through sdv_ba_get_system (HA, bA, Hsc, bsc slots).
 * sdv_ba_marginalize_frame EnergyFunctional::marginalizeFrame, EnergyFunctional.cpp:434-512: Schur-eliminates frame idx from (HM,bM) and drops it
 *                          from the window; points/residuals must be re-set (sdv_ba_set_points) before the window is used again.
 * sdv_ba_get_prior         reads (HM,bM) of the current window, dim = 4 + 6*nF (row-major). */
int  sdv_ba_flag_points(sdv_ctx* c, const int32_t* selected, int32_t* status_out);
int  sdv_ba_marginalize_points(sdv_ctx* c, const int32_t* status);
int  sdv_ba_marginalize_frame(sdv_ctx* c, int idx);
int  sdv_ba_get_prior(sdv_ctx* c, int* dim, double* HM, double* bM);
/* ---- batched install and hand-over: the per-window entries above for n windows of one context in one call each (FullSystem::makeKeyFrame around
 * optimize, FullSystem.cpp:1152-1171, for every resident sequence).  Windows are named by index (sdv_ba_select numbering), each at most once; every
 * per-window array is the call's arrays concatenated in the order the windows are listed.  The number of launches and host waits of a call does not
 * grow with n (sdv_launch_count, sdv_ba_host_wait_count).  A refused call (SDV_ERR_ARG, the message names the window and the point or residual) leaves
 * every listed window as it was, and so does a failed allocation; a CUDA error in the launches themselves leaves the listed windows undefined.
 * sdv_ba_set_window_batch        insertFrame + setAdjointsF + the HM/bM carry-over (sdv_ba_set_window) and CalibHessian::value_zero (sdv_ba_set_calib_zero)
 *                                for n windows.  Window i holds frames f_begin[i] .. f_begin[i+1] (1..SDV_MAX_FRAMES_WINDOW, one size); the per-frame
 *                                arrays are indexed by that frame range; calib_value_scaled[4n], calib_value_zero[4n] (NULL: value_zero = value);
 *                                HM / bM (NULL: zero) concatenated per window with dim = 4 + 6 nF_i.  A window not set before is created.
 *                                A window gets its point storage at its first sdv_ba_set_points(_batch), zero points included.
 * sdv_ba_set_points_batch        makeIDX + setPrecalcValues (sdv_ba_set_points) for n windows: window i's points are p_begin[i] .. p_begin[i+1], its
 *                                residuals r_begin[i] .. r_begin[i+1]; res_begin and r_point are window-local, window i's res_begin block has nP_i + 1
 *                                entries and starts at p_begin[i] + i.  The checks run on the device before any window changes.
 * sdv_ba_flag_points_batch       sdv_ba_flag_points for n windows; selected / status_out concatenated by the windows' point counts.
 * sdv_ba_marginalize_points_batch sdv_ba_marginalize_points for n windows; status NULL: each window's device-resident status of the flag call.
 * sdv_ba_marginalize_frames_batch EnergyFunctional::marginalizeFrame, repeated: window i eliminates frames idx[k_begin[i] .. k_begin[i+1]) in that order,
 *                                each index into the window as the previous eliminations left it (the reference's `i = 0` restart); zero frames is
 *                                allowed, elimination down to zero frames is refused.  HM_out / bM_out (may be NULL) receive every window's prior
 *                                afterwards, concatenated, dim = 4 + 6 nF_i.  Unpinning and the stale-points rule are those of sdv_ba_marginalize_frame. */
int  sdv_ba_set_window_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* f_begin, const uint64_t* frame_ids, const double* T_evalPT7,
                             const double* state10, const double* state_zero10, const float* ab_exposure, const int32_t* frameID, const float* frameEnergyTH,
                             const double* calib_value_scaled, const double* calib_value_zero, const double* HM, const double* bM);
int  sdv_ba_set_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* p_begin, const int32_t* r_begin, const float* uv, const float* idepth,
                             const float* idepth_zero, const float* color8, const float* weights8, const int32_t* host, const int32_t* hasDepthPrior,
                             const int32_t* isFromSensor, const int32_t* res_begin, const int32_t* r_point, const int32_t* r_host, const int32_t* r_target,
                             const int32_t* r_hasMatcher, const float* r_matcher, const int32_t* r_isNew);
/* host waits on the back-end stream so far (each synchronise of an sdv_ba_* entry, and the wait of a staging buffer that grows) */
long long sdv_ba_host_wait_count(sdv_ctx* c);
int  sdv_ba_flag_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* selected, int32_t* status_out);
int  sdv_ba_marginalize_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* status);
int  sdv_ba_marginalize_frames_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* k_begin, const int32_t* idx, double* HM_out, double* bM_out);
int  sdv_ba_get_linearized(sdv_ctx* c, float* res_toZero2, int32_t* isLinearized);
int  sdv_ba_get_system(sdv_ctx* c, double* HA, double* bA, double* Hsc, double* bsc, double* lastHS, double* lastbS);
int  sdv_ba_get_precalc(sdv_ctx* c, int host, int target, float out27[27], double adHost36[36], double adTarget36[36], float adHTdelta6[6]);

/* =====================================================================================================================
 * Candidate management at keyframe rate (SURVEY.md §8f rank 4 and the caller half of rank 2).  Tracker call domain.
 *   PixelSelector                         FullSystem/PixelSelector2.cpp:11-26 (ctor), :47-106 makeHists, :354-622 makeMapsFromLidar / selectFromLidar,
 *                                         :108-352 makeMaps / select
 *   FullSystem::makeNewTraces             FullSystem/FullSystem.cpp:1273-1356 (+ shiTomasiScore :1540-1583, setMask :1261-1271, ImmaturePoint ctor)
 *   CoarseDistanceMap, activatePointsMT   FullSystem/CoarseTracker.cpp:1139-1282, FullSystem/FullSystem.cpp:600-671
 * A selector SLOT stands for one PixelSelector / FullSystem::selectionMap pair, i.e. one resident sequence: it carries currentPotential (initially 3) and the
 * persistent monocular selection map (w*h bytes, values 0 / 1 / 2 / 4 — the reference's float map; zero at birth where the reference's is uninitialised).
 * random_pattern: the w*h bytes of PixelSelector::randomPattern — the caller generates them exactly like the constructor does (srand(3141592); rand() & 0xFF), so the
 * library never touches the process-wide rand() stream.  Reads of thsSmoothed past its (h/32) rows — the reference indexes its uninitialised tail for the last
 * image rows — see zeros here.  LiDAR pixels are rows {Ku, Kv, depth} of doubles, as main.cpp:810-848 pushes them into FullSystem::qCloudPixel.
 * Cameras of another size (sdv_set_camera_size): sdv_selector_set_slot_cams binds slot slots[i] to camera cams[i] (after sdv_selector_init every slot is on
 * camera 0).  A slot on camera c works at w_c x h_c: its frames must have that size (else SDV_ERR_ARG), its persistent map is w_c*h_c bytes
 * (sdv_selector_get_map), and its pattern is the first w_c*h_c bytes of random_pattern (what PixelSelector(w_c, h_c) draws after the same srand).  Rebinding
 * a slot to a camera of another size starts it afresh (map zeroed, currentPotential 3: a new PixelSelector); the same size keeps its state.  A slot or
 * camera out of range returns SDV_ERR_ARG and changes no slot.  sdv_selector_make_hists_cam: the frame is camera cam's ((w_c/32) x (h_c/32) blocks). */
typedef struct { float u, v, my_type, score, idepth_fromSensor; int32_t isFromSensor, type; } sdv_new_trace;   /* type: 0 CORNER, 1 EDGELET (ImmaturePoint.h), -1 not assigned (monocular points) */
int  sdv_selector_init(sdv_ctx* c, const uint8_t* random_pattern, int n_slots);
int  sdv_selector_potential(sdv_ctx* c, int slot, int set_to /* <= 0: leave */, int* out);
int  sdv_selector_get_map(sdv_ctx* c, int slot, uint8_t* out_wh);
int  sdv_selector_set_slot_cams(sdv_ctx* c, int n, const int32_t* slots, const int32_t* cams);
/* The running LiDAR pixel box FullSystem::left, right, up, down (FullSystem.h:191-194) belongs to the sequence, like selectionMap: every selector slot keeps
 * one on the device.  It is {10000, -1, 10000, -1} when the slot is created (sdv_selector_init) and whenever a rebind to a camera of another size starts the
 * slot afresh; sdv_lidar_handler_rows_batch reads and updates it.  set_to (may be NULL: leave) writes it, stream-ordered after the handler calls enqueued
 * so far (a mid-drive start); lrud_out (may be NULL) reads it back, waiting for those calls.  A slot out of range returns SDV_ERR_ARG. */
int  sdv_selector_lidar_box(sdv_ctx* c, int slot, const int32_t* set_to, int32_t* lrud_out);
/* void PixelSelector::makeHists(const FrameHessian*): ths / thsSmoothed of the (w/32) x (h/32) blocks */
int  sdv_selector_make_hists(sdv_ctx* c, uint64_t frame, float* ths_out, float* thsSmoothed_out);
int  sdv_selector_make_hists_cam(sdv_ctx* c, int cam, uint64_t frame, float* ths_out, float* thsSmoothed_out);
/* int PixelSelector::makeMapsFromLidar(fh, map_out, density, recursionsLeft, plot, thFactor, vCloudPixel) for n (slot, frame) pairs at once when cloud_begin != NULL
 * (job j owns cloud rows cloud_begin[j] .. cloud_begin[j+1]; maps_out = the n maps back to back, one byte per cloud row), and
 * int PixelSelector::makeMaps(fh, map_out, density, recursionsLeft, plot, thFactor) when cloud_begin == NULL (maps_out = the n maps back to back, job j's at its slot's
 * camera size w_c*h_c; the slot's persistent map is the one written).  makeHists runs first, like `if(fh != gradHistFrame) makeHists(fh)`.  num_have_out[j] = the return value; the slot's currentPotential is updated. */
int  sdv_selector_make_maps_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density,
                                  const int32_t* recursions_left, const float* th_factor, uint8_t* maps_out, int32_t* num_have_out);
/* void FullSystem::makeNewTraces(FrameHessian* newFrame, float*) for n new keyframes (one per sequence / slot) in one call.  density_lidar[j] =
 * ((float)lidarArea/(float)imageArea) * setting_desiredImmatureDensity (:1287-1290), density_dense[j] = setting_desiredImmatureDensity (:1293), add_feature_point[j] =
 * FullSystem::addFeaturePoint (off: the slot's map of an EARLIER keyframe is walked again, as in the reference).  Per job up to `cap` points come back in creation order
 * (LiDAR points in cloud order, then monocular points in raster order): out[j*cap ..] and, if imm_out != NULL, the constructed ImmaturePoint records imm_out[j*cap ..];
 * n_out[j] = how many; num_points2[2j..] = {numPointLidar, numPointMonocular}.  SDV_ERR_CAPACITY when cap is too small. */
int  sdv_make_new_traces_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density_lidar,
                               const float* density_dense, const int32_t* add_feature_point, int cap, sdv_new_trace* out, sdv_immature_pt* imm_out, int32_t* n_out, int32_t* num_points2);
/* The same with the points deposited into the immature-point store (sdv_immature_store_set) instead of returned: job j's points, in creation order, replace the block of
 * frames[j], with what the host does around the call in the reference applied on the device — for LiDAR points idepth_fromSensor = 1.0/depth and
 * idepth_min = idepth_max = idepth_fromSensor (FullSystem.cpp:1313-1317), lastTraceStatus = IPS_SKIPPED (makeKeyFrame, :1080-1084); meta = {my_type, type, isFromSensor,
 * idepth_fromSensor} of the sdv_new_trace record.  n_out / num_points2 as above; cap bounds the points of a job as above.  A frame named twice returns SDV_ERR_ARG. */
int  sdv_make_new_traces_store_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density_lidar,
                                     const float* density_dense, const int32_t* add_feature_point, int cap, int32_t* n_out, int32_t* num_points2);
/* FullSystem::makeNewTraces (FullSystem.cpp:1273-1356) fed from the LiDAR row sets (sdv_lidar_handler_rows_batch): sdv_make_new_traces_store_batch with job j's rows,
 * box and flag taken from frames[j]'s row set, which never leaves the device — density_lidar = ((float)((right-left)*(down-up)) / (float)(w_c*h_c)) * desired_density[j]
 * from the set's box and the slot camera's size (:1287-1290), density_dense = desired_density[j], add_feature_point = the set's addFeaturePoint.  Outputs and rules
 * as sdv_make_new_traces_store_batch.  A frame without a row set returns SDV_ERR_NOFRAME, an overflowed set SDV_ERR_CAPACITY; either way no block and no selector
 * state changes.  The call waits for the device (the potential adaptation runs on the host), after reading every job's header in one copy.
 * Difference from the reference: there, addFeaturePoint and the box are whatever the LATEST lidarCloudHandler left; here they are the snapshot taken with frames[j]'s
 * sweep.  The two agree whenever a frame's keyframe work runs before the next sweep is handled — the sequential order of process() (main.cpp:470-508), and what
 * the host-row path gives. */
int  sdv_make_new_traces_rows_store_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const float* desired_density, int cap, int32_t* n_out,
                                          int32_t* num_points2);
/* The start of a sequence (FullSystem::addActiveFrame for frames 0 and 1 of a LiDAR run, FullSystem.cpp:842-850 and :299-338), for n sequences in one call.  Job j
 * bootstraps keyframe frames[j] on tracker slot slots[j], at the size and depth of that slot's camera (sdv_set_calib_slots_cams):
 *   CoarseInitializer::setFirstFromLidar, level 0 (CoarseInitializer.cpp:766-888): a FRESH PixelSelector (currentPotential 3, makeHists, the camera's prefix of the
 *     random pattern) runs makeMapsFromLidar(frame, statusMap, 0.03f*lidarArea, 1, false, 2, rows), lidarArea = (right-left)*(down-up) of the box; the Pnt list
 *     is the rows with status != 0 and (float)depth > 0 in cloud order.  No selector slot is read or written (potential, map and box stay as they are).
 *   FullSystem::initializeFromInitializer's point loop (FullSystem.cpp:1176-1225): Pnt k is dropped when rand_draws[draw_begin[j] + k] / (float)RAND_MAX >
 *     desired_point_density[j] / numPoints[0] (rand_draws: the C library's rand() values, glibc RAND_MAX), else it becomes ImmaturePoint((int)(u+0.5f),
 *     (int)(v+0.5f)) with idepth_min = idepth_max = 1/depth and, when its energyTH is finite, a PointHessian with idepth = idepth_zero = 1/depth, hasDepthPrior,
 *     ACTIVE and isFromSensor.  n_selected_out[j] = numPoints[0]: the caller's rand() stream moves on by that much.  n_out[j] = the points kept; for each, in Pnt
 *     order, the sdv_immature_pt record pts_out[j*cap + i], sdv_immature_meta meta_out[j*cap + i] = {my_type = status byte, type 0 CORNER, isFromSensor 1,
 *     idepth_fromSensor = 1/depth} and idepth_out[j*cap + i] = the PointHessian's idepth and idepth_zero (each of the three may be NULL).
 *   CoarseTracker::setCTRefForFirstFrame (CoarseTracker.cpp:636-647, :108-256): tracker slot slots[j] gets the reference of sdv_tracker_set_ref with the splat rows
 *     {u, v, idepth, HdiF 0}, round_half 1, ref_frame = frames[j], ref_a = ref_b = 0; and map slot slots[j] gets sdv_map_set of one keyframe frames[j] with identity
 *     camToWorld, aff_g2l {0, 0} and the kept points {u, v, idepth, host 0, CORNER}.  No record crosses PCIe for this.
 * Reference behaviour restated: EFPoint::HdiF is read uninitialised by makeCoarseDepthForFirstFrame (taken as 0, a zeroed block) and PointHessian::type is never set
 * for these points (taken as CORNER).  A point whose 8-pattern would read outside the frame's plane is not kept (the reference reads past its image there).
 * job j has rows cloud3[3*cloud_begin[j] ..] (host, cloud_begin[0] = 0) and box lrud[4j..] = FullSystem::left, right, up, down after its sweep; the _rows form takes
 * both from frames[j]'s row set (sdv_lidar_handler_rows_batch).  Refused before anything is enqueued, changing no slot: sdv_selector_init missing (SDV_ERR_STATE);
 * a frame without a row set (SDV_ERR_NOFRAME) or with an overflowed one (SDV_ERR_CAPACITY); fewer draws than rows, a slot out of range or named twice, a frame
 * named twice, a slot camera of fewer than 3 levels (SDV_ERR_ARG); a frame of another size than its slot's camera (as sdv_tracker_set_ref).  More than cap kept
 * points in a job return SDV_ERR_CAPACITY with n_out and n_selected_out filled and no slot changed.  A reference cloud over max_ref_points behaves as in
 * sdv_tracker_set_ref.  An empty cloud keeps no point: the slot's reference has 0 points at every level.  The call waits for the device. */
int  sdv_init_from_lidar_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const int32_t* lrud,
                               const float* desired_point_density, const int32_t* draw_begin, const int32_t* rand_draws, int cap, int32_t* n_out, int32_t* n_selected_out,
                               sdv_immature_pt* pts_out, sdv_immature_meta* meta_out, float* idepth_out);
int  sdv_init_from_lidar_rows_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const float* desired_point_density, const int32_t* draw_begin,
                                    const int32_t* rand_draws, int cap, int32_t* n_out, int32_t* n_selected_out, sdv_immature_pt* pts_out, sdv_immature_meta* meta_out,
                                    float* idepth_out);
/* The selection half of void FullSystem::activatePointsMT() for n sequences: CoarseDistanceMap::makeDistanceMap from the ACTIVE points of the other keyframes, then the
 * candidate walk :600-671 with addIntoDistFinal after every accept.  Sequence j owns source keyframes host_begin[j] .. host_begin[j+1] (their points: uvid rows
 * pt_begin[k] .. pt_begin[k+1] = {u, v, idepth_scaled}; KRKi9 / Kt3 per keyframe = K[1] R K[0]^-1, K[1] t of host -> newest, FullSystem.cpp:606-608) and candidate
 * keyframes cand_host_begin[j] .. (their candidates: cand4 rows {u, v, 0.5f*(idepth_max+idepth_min), my_type} that passed the deletion / canActivate tests of
 * :618-645, which are pointer-graph bookkeeping).  decision_out per candidate: 1 = handed to optimizeImmaturePoint (sdv_immature_optimize_batch), 0 = too close to
 * existing points, -1 = projects outside the level-1 image (deleted).  dist_map_out (optional): n maps of (w/2)*(h/2) floats = fwdWarpedIDDistFinal after the walk.
 * _cams: sequence j is camera cams[j]'s, its map and walk are at (w_c/2) x (h_c/2) and dist_map_out holds the maps back to back, each at its own size;
 * cams == NULL is sdv_activate_select_batch (camera 0). */
int  sdv_activate_select_batch(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                               const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4, const float* min_act_dist,
                               int32_t* decision_out, float* dist_map_out);
int  sdv_activate_select_batch_cams(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                                    const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4,
                                    const float* min_act_dist, const int32_t* cams, int32_t* decision_out, float* dist_map_out);

/* =====================================================================================================================
 * LiDAR front-end of the node (SURVEY.md §8f rank 3, second half): void lidarCloudHandler(const sensor_msgs::PointCloud2ConstPtr&)   src/main.cpp:785-858
 *   -> projectPointCloud :563-607, groundRemoval :609-655, cloudSegmentation / labelComponents :657-783, projection into the image :806-849.  Tracker call domain.
 * sdv_lidar_init: the sensor constants of main.cpp:103-108 (N_SCAN, Horizon_SCAN, ang_res_x, ang_res_y, ang_bottom, groundScanInd; Velodyne-64: 64, 1800, 0.2, 0.427, 24.9, 50).
 * sdv_lidar_handler_batch: n raw sweeps (one per resident sequence), sweep j = XYZI rows sweep_begin[j] .. sweep_begin[j+1] of xyzi (the decoded PointCloud2, what
 * pcl::fromROSMsg yields; rows with a non-finite coordinate are dropped like pcl::removeNaNFromPointCloud does).  Per sweep: Rlc9 (row-major) / tlc3 = FullSystem::Rlc, tlc
 * (LiDAR -> camera), K4 = FullSystem::fx fy cx cy, lrud_io = FullSystem::left, right, up, down (the running pixel box; 10000, -1, 10000, -1 at start).  The image
 * size, which bounds the pixel box, is camera 0's (the context's); sdv_lidar_handler_batch_cams takes it from camera cams[j] for sweep j.  Out, per sweep: up to cap rows {Ku, Kv, depth} (doubles, the vCloudPixel pushed into FullSystem::qCloudPixel, same order) at
 * cloud3_out[3*j*cap ..], n_out[j] rows, add_feature_point_out[j] = FullSystem::addFeaturePoint (ground ratio > 0.8), stats_out[2j..] = {numGround, size of
 * segmentedCloud} (may be NULL).  The rows feed sdv_make_new_traces_batch and the LiDAR-depth splats of sdv_tracker_set_ref. */
int  sdv_lidar_init(sdv_ctx* c, int n_scan, int horizon_scan, float ang_res_x, float ang_res_y, float ang_bottom, int ground_scan_ind);
int  sdv_lidar_handler_batch(sdv_ctx* c, int n, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9, const double* tlc3, const float* K4, int32_t* lrud_io, int cap,
                             double* cloud3_out, int32_t* n_out, int32_t* add_feature_point_out, int32_t* stats_out);
int  sdv_lidar_handler_batch_cams(sdv_ctx* c, int n, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9, const double* tlc3, const float* K4, const int32_t* cams,
                                  int32_t* lrud_io, int cap, double* cloud3_out, int32_t* n_out, int32_t* add_feature_point_out, int32_t* stats_out);
/* Row sets: FullSystem::qCloudPixel on the device, keyed by frame handle.  lidarCloudHandler (main.cpp:785-858) pushes a sweep's rows, process() pairs the front
 * image with the front cloud and pops both after addActiveFrame (main.cpp:470-508); keying the rows by the handle the paired image gets makes that pairing
 * explicit and lets a sweep be ingested ahead of its image (the frame need not be resident).  A set holds up to its deposit's cap rows {Ku, Kv, depth} (doubles,
 * the reference's order) and a header: the true row count (also past cap), an overflow mark, the running box {left, right, up, down} as it stood after this
 * sweep, addFeaturePoint, numGround and the size of segmentedCloud.  A deposit under an existing handle replaces its set.  Blocks are reused in place when the
 * new cap fits, else a spare or a new allocation with headroom is taken; dropped sets become spares.  Tracker call domain.
 * sdv_lidar_handler_rows_batch: the handler of sdv_lidar_handler_batch_cams writing into row sets.  Sweep j belongs to the sequence on selector slot slots[j]: its
 * camera is the slot's (its size bounds the box, main.cpp:828), the box is the slot's (sdv_selector_lidar_box) and is updated on the device, the rows go into
 * frames[j]'s set.  Refused before anything is enqueued, changing nothing: sdv_lidar_init or sdv_selector_init missing (SDV_ERR_STATE); a slot out of range,
 * a slot or a frame named twice, cap < 1 (SDV_ERR_ARG).  Without stats_out the call enqueues and returns: the sweep upload goes on the copy stream, so it
 * overlaps tracking already enqueued, and the kernels wait for it by event.  Pinned xyzi must stay valid until the next call that synchronises (as for the image
 * uploads).  With stats_out it waits and fills {rows, numGround, n_segmented, addFeaturePoint, overflow} per sweep.  More rows than cap keep the true count in
 * the header and mark the set; nothing is written past cap, and every consumer of the set returns SDV_ERR_CAPACITY.
 * sdv_lidar_rows_get: frame's rows (cap: room in cloud3_out; cloud3_out NULL: header only), *n_out = the true count, the box and the flag; waits.
 * sdv_lidar_rows_drop: qCloudPixel.pop() (main.cpp:507) for n frames.  A handle without a set returns SDV_ERR_NOFRAME from both and changes nothing. */
int  sdv_lidar_handler_rows_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9,
                                  const double* tlc3, const float* K4, int cap, int32_t* stats_out);
int  sdv_lidar_rows_get(sdv_ctx* c, uint64_t frame, int cap, double* cloud3_out, int32_t* n_out, int32_t* lrud_out, int32_t* add_feature_point_out);
int  sdv_lidar_rows_drop(sdv_ctx* c, int n, const uint64_t* frames);

#ifdef __cplusplus
}
#endif
#endif /* SDV_B200_H */
