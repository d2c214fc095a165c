// sdv_refine.cuh — job descriptor of the structPoseEstimation kernel (sdv_refine.cu), shared with the fused per-frame refinement
// (sdv_reproject.cu: reprojectMap -> structPoseEstimation without leaving the device).
#pragma once
#include <cuda_runtime.h>
#include "sdv_device.cuh"
#include "../../include/sdv_b200.h"

namespace sdv {

struct RefineJob {
  double T[7];                           // curToWorld in/out
  const double* hostT;                   // camToWorld of the job's host keyframes (7 doubles each) or nullptr -> hostT7 + 7*host_begin of the launch
  int pt_begin, pt_end, host_begin, nH;
  int geom_row;                          // row of the geometry table: the K of the tracker slot the job belongs to
  float res; int iterations, accepts, num;
};

cudaError_t refine_init_device();
void launch_struct_pose(RefineJob* jobs, int n_jobs, const sdv_overlap_pt* pts, const double* hostT7, const GeomRow* geom_tab, cudaStream_t st);

} // namespace sdv
