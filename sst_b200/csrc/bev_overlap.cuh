// The rotated bird's-eye-view overlap of two [x1, y1, x2, y2, r] boxes (see iou3d.cu for the geometry), shared by the IoU / NMS
// kernels of iou3d.cu and the 3-D IoU of roi_head.cu's assignment, so both compute the same fp32 area.
#pragma once
#include "common.cuh"

namespace {

struct BevBox {
  float x1, y1, x2, y2;  // raw corners (the centre offset of two boxes is formed from their differences)
  float hx, hy;          // half extents (|.|: a box given with x2 < x1 has the same corner set)
  float c, s;            // cos r, sin r
  float rad2;            // squared circumradius
  float area;            // (x2 - x1)(y2 - y1), the reference's area
};

__device__ __forceinline__ BevBox make_bev(const float* __restrict__ p) {
  BevBox b;
  b.x1 = p[0];
  b.y1 = p[1];
  b.x2 = p[2];
  b.y2 = p[3];
  b.hx = 0.5f * fabsf(b.x2 - b.x1);
  b.hy = 0.5f * fabsf(b.y2 - b.y1);
  sincosf(p[4], &b.s, &b.c);
  b.rad2 = b.hx * b.hx + b.hy * b.hy;
  b.area = (b.x2 - b.x1) * (b.y2 - b.y1);
  return b;
}

// Shoelace accumulator at the end of the clipping pipeline.
struct AreaSink {
  float fx, fy, px, py, sum;
  int n;
  __device__ __forceinline__ void put(float x, float y) {
    if (n == 0) {
      fx = x;
      fy = y;
    } else {
      sum += px * y - py * x;
    }
    px = x;
    py = y;
    n++;
  }
  __device__ __forceinline__ void close() {
    if (n > 0) sum += px * fy - py * fx;
  }
};

// One Sutherland-Hodgman stage: keeps SG * (AX ? y : x) <= h.  Vertices stream through put(); close() feeds the closing edge.
template <int AX, int SG, typename Next>
struct ClipStage {
  Next& next;
  float h;
  float fx, fy, fd, px, py, pd;
  bool has;
  __device__ __forceinline__ ClipStage(Next& nx, float hh) : next(nx), h(hh), fx(0), fy(0), fd(0), px(0), py(0), pd(0), has(false) {}
  __device__ __forceinline__ void cross(float ax, float ay, float ad, float bx, float by, float bd) {
    const float t = ad / (ad - bd);  // ad and bd lie on opposite sides of 0, so the denominator is not 0
    if (AX == 0) next.put((float)SG * h, ay + t * (by - ay));
    else next.put(ax + t * (bx - ax), (float)SG * h);
  }
  __device__ __forceinline__ void put(float x, float y) {
    const float d = (float)SG * (AX == 0 ? x : y) - h;
    if (!has) {
      fx = x;
      fy = y;
      fd = d;
      has = true;
    } else if ((pd <= 0.f) != (d <= 0.f)) {
      cross(px, py, pd, x, y, d);
    }
    if (d <= 0.f) next.put(x, y);
    px = x;
    py = y;
    pd = d;
  }
  __device__ __forceinline__ void close() {
    if (has && (pd <= 0.f) != (fd <= 0.f)) cross(px, py, pd, fx, fy, fd);
    next.close();
  }
};

__device__ __forceinline__ float bev_overlap(const BevBox& a, const BevBox& b) {
  // centre of b relative to a: differences of nearby coordinates are exact, their half-sum rounds once
  const float dx = 0.5f * ((b.x1 - a.x1) + (b.x2 - a.x2)), dy = 0.5f * ((b.y1 - a.y1) + (b.y2 - a.y2));
  const float rr = a.rad2 + b.rad2 + 2.f * sqrtf(a.rad2 * b.rad2);  // (Ra + Rb)^2
  if (dx * dx + dy * dy > rr || a.hx * a.hy == 0.f || b.hx * b.hy == 0.f) return 0.f;  // apart, or a zero-area box
  // into a's frame: local = R(ra) * world; b is turned by t = ra - rb there
  const float cx = dx * a.c - dy * a.s, cy = dx * a.s + dy * a.c;
  const float ct = a.c * b.c + a.s * b.s, st = a.s * b.c - a.c * b.s;
  const float ux = ct * b.hx, uy = st * b.hx;    // b's half side along its local x
  const float vx = -st * b.hy, vy = ct * b.hy;   // ... and along its local y
  AreaSink sink{0.f, 0.f, 0.f, 0.f, 0.f, 0};
  ClipStage<1, -1, AreaSink> s3(sink, a.hy);
  ClipStage<1, 1, ClipStage<1, -1, AreaSink>> s2(s3, a.hy);
  ClipStage<0, -1, ClipStage<1, 1, ClipStage<1, -1, AreaSink>>> s1(s2, a.hx);
  ClipStage<0, 1, ClipStage<0, -1, ClipStage<1, 1, ClipStage<1, -1, AreaSink>>>> s0(s1, a.hx);
  s0.put(cx - ux - vx, cy - uy - vy);
  s0.put(cx + ux - vx, cy + uy - vy);
  s0.put(cx + ux + vx, cy + uy + vy);
  s0.put(cx - ux + vx, cy - uy + vy);
  s0.close();
  return 0.5f * fabsf(sink.sum);
}

}  // namespace
