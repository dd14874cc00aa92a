// Point-in-box test of mmdet3d's roiaware_pool3d package: the arithmetic of check_pt_in_box3d
// (mmdet3d/ops/roiaware_pool3d/src/points_in_boxes_cuda.cu:24-49), evaluated as the same float expressions: centre z = bottom + h/2 in
// double, |z - cz| > h/2 rejects, angle rz + pi/2 formed in double, cos / sin in float, local x / y as (sx cos - sy sin, sx sin + sy cos)
// rounded as the reference kernel rounds them, strict |local| < l/2, w/2.  Shared by box3d.cuh (roi_pool.cu, roiaware.cu), voteseg.cu
// and cluster_head.cu, so every hit is bit-identical to the reference's points_in_boxes_gpu.
#pragma once
#include "common.cuh"

namespace {

struct Box {
  float cx, cy, ca, sa;  // centre, cos / sin of rz + pi/2
  float cz, hl, hw, hh;  // centre z, half l / w / h
};

__device__ __forceinline__ Box make_box(float cx, float cy, float zb, float w, float l, float h, float rz) {
  Box b;
  b.cx = cx;
  b.cy = cy;
  b.cz = (float)((double)zb + (double)h / 2.0);
  const float ang = (float)((double)rz + M_PI / 2.0);
  b.ca = cosf(ang);
  b.sa = sinf(ang);
  b.hl = 0.5f * l;
  b.hw = 0.5f * w;
  b.hh = 0.5f * h;
  return b;
}

// The reference's `sx * cos + sy * (-sin)` / `sx * sin + sy * cos` compiles (nvcc, sm_90a, default contraction) to the product with cos
// fused and the one with sin rounded first; left to itself the compiler contracts this file's copy the other way for local y, so the
// rounding is spelled out.
__device__ __forceinline__ void to_local(const Box& b, float x, float y, float& lx, float& ly) {
  const float sx = x - b.cx, sy = y - b.cy;
  lx = __fmaf_rn(sx, b.ca, __fmul_rn(sy, -b.sa));
  ly = __fmaf_rn(sy, b.ca, __fmul_rn(sx, b.sa));
}

__device__ __forceinline__ bool in_box(const Box& b, float z, float lx, float ly) {
  return !(fabsf(z - b.cz) > b.hh) && lx > -b.hl && lx < b.hl && ly > -b.hw && ly < b.hw;
}

}  // namespace
