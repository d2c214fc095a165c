// sdv_kernels.cuh — launcher declarations (host side of sdv_kernels.cu / sdv_ba_kernels.cu)
#pragma once
#include "sdv_device.cuh"
#include "../../include/sdv_b200.h"

namespace sdv {

// pyramid (FrameHessian::makeImages, HessianBlocks.cpp:107-167)
struct PyrBatchHost { const void* src; float* I0; float* pyr; int flags; int cam; int w, h; };   // mirrors PyrBatch in sdv_kernels.cu
// geometric + photometric undistortion tables of the ingest (util/Undistort.cpp): device pointers; G / vignette may be null
struct UndistortDev { const float* remapX; const float* remapY; const float* G; const float* vignette; int wOrg, hOrg; float factor; };
// the cameras of a context (sdv_set_undistort_cam), passed by value to the RAW kernels; an unset camera has remapX == nullptr
struct UndistortCams { UndistortDev cam[SDV_MAX_CAMERAS]; };
// all planes of levels >= 1 in one launch (levels > 1); each frame has its own size PyrBatch::w x h, and its `pyr` holds level l after levels 1..l-1 of
// that size; max_w x max_h: the largest frame of the batch (grid and shared memory); vec: 16-byte aligned inputs / I0 and w % 4 == 0 for every frame.
// und: RAW input, each frame rectified with und->cam[PyrBatch::cam]
void launch_pyramid_batch(const void* batch_dev, int nframes, bool src_u8, bool vec, int max_w, int max_h, int levels, cudaStream_t st, const UndistortCams* und = nullptr);
void launch_pyramid_copy0(const void* batch_dev, int nframes, bool src_u8, int max_w, int max_h, cudaStream_t st, const UndistortCams* und = nullptr);
void launch_grad_texels(const float* I, float4* out, int w, int h, const float* gw2, cudaStream_t st);   // packed {I,dx,dy,|grad|^2} texels of one planar level (gw2: gamma_w2)
void launch_unpack_level(const float4* in, float* dI3, float* ab, int n, cudaStream_t st);

cudaError_t kernels_init_device();        // per-device function attributes of the tracker kernels (called by sdv_create after cudaSetDevice)
// fused calcRes + calcGSSSE, one launch (CoarseTracker.cpp:486-634, 427-484)
int  step_kernel_max_grid();
void launch_coarse_res_gs(const float4* pts, int n, const float* I, const LevelGeom& g, const EvalParams& ep,
                          double* partials, unsigned int* ticket, double* totals, cudaStream_t st);

// device-resident trackNewestCoarse (CoarseTracker.cpp:662-838): njobs clusters of cluster_size CTAs
// small host->device transfer done by a kernel reading pinned (UVA-mapped) host memory: it does not queue behind bulk cudaMemcpyAsync traffic on the
// H2D copy engine, so a job-descriptor upload cannot be delayed by the next batch's image upload (DESIGN.md §6)
void launch_h2d_words(void* dst_dev, const void* src_pinned, size_t bytes, cudaStream_t st);
cudaError_t launch_track_cluster(TrackJob* jobs_dev, int njobs, const TrackConst* tc_dev, const GeomRow* geom_dev, int cluster_size, int threads, cudaStream_t st);

void launch_pack_cloud(const float* u, const float* v, const float* id, const float* col, int n, float4* out, cudaStream_t st);

} // namespace sdv
