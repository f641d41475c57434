// The rotated BEV overlap of two boxes, shared by the NMS / IoU kernels (box_nms.cu) and the TransFusion
// assignment cost (transfusion_assign.cu).  Internal header.
//
// Boxes are [x1, y1, x2, y2, ry] fp32.  A box is the axis-aligned extent turned by ry about its centre:
//   x' = (x - cx) cos r + (y - cy) sin r + cx,   y' = -(x - cx) sin r + (y - cy) cos r + cy.
// The overlap is the area of the convex intersection polygon, whose vertices are the strict edge crossings
// (both segments cut strictly) and the corners of each box that lie inside the other one within 1e-5 (tested in
// the other box's own frame), ordered by pseudo-angle about their mean and summed as a triangle fan.
#pragma once
#include "common.cuh"

namespace bevb200 {
namespace {

constexpr float kInsideMargin = 1e-5f;
// Vertex buffer of the intersection polygon.  Two convex quadrilaterals meet in at most 8 edge crossings plus 8
// corners; the pushes are guarded anyway, so rounding in a near-degenerate pair can never write past the buffer.
constexpr int kMaxVertices = 16;

struct RotBox {
  float cx, cy, hx, hy, c, s;   // centre, half extents, cos / sin of ry
};

__device__ __forceinline__ RotBox load_rot(const float *b) {
  RotBox r;
  r.cx = (b[0] + b[2]) * 0.5f;
  r.cy = (b[1] + b[3]) * 0.5f;
  r.hx = (b[2] - b[0]) * 0.5f;
  r.hy = (b[3] - b[1]) * 0.5f;
  sincosf(b[4], &r.s, &r.c);
  return r;
}

__device__ __forceinline__ float cross2(float ax, float ay, float bx, float by) { return ax * by - ay * bx; }

// Corners (x1, y1), (x2, y1), (x2, y2), (x1, y2) turned about the centre, relative to the point (ox, oy).
__device__ __forceinline__ void corners(const RotBox &b, float ox, float oy, float2 (&p)[4]) {
  const float px = b.cx - ox, py = b.cy - oy;
  const float xs[4] = {-b.hx, b.hx, b.hx, -b.hx}, ys[4] = {-b.hy, -b.hy, b.hy, b.hy};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    p[k] = make_float2(xs[k] * b.c + ys[k] * b.s + px, -xs[k] * b.s + ys[k] * b.c + py);
}

// p (relative to (ox, oy)) inside b within the margin, p turned back by -r about b's centre.  NaN gives false.
__device__ __forceinline__ bool inside(const RotBox &b, float ox, float oy, float2 p) {
  const float dx = p.x - (b.cx - ox), dy = p.y - (b.cy - oy);
  const float rx = dx * b.c - dy * b.s, ry = dx * b.s + dy * b.c;
  return rx > -b.hx - kInsideMargin && rx < b.hx + kInsideMargin && ry > -b.hy - kInsideMargin &&
         ry < b.hy + kInsideMargin;
}

// Position of the direction (dx, dy) on [0, 4), monotone in atan2 over one turn.
__device__ __forceinline__ float pseudo_angle(float dx, float dy) {
  const float t = fabsf(dx) + fabsf(dy);
  const float p = t > 0.f ? dx / t : 1.f;
  return dy >= 0.f ? 1.f - p : 3.f + p;
}

// The polygon is built relative to a's centre, so its vertices carry the rounding of the box sizes rather
// than of the absolute positions (up to 61 m in the CenterHead range).
__device__ float rot_overlap(const RotBox &a, const RotBox &b) {
  // Conservative early-out: circumscribed circles apart by a relative 1e-3 plus 1e-3 leave no vertex
  // (the full evaluation would also give 0).  NaN compares false and takes the full path.
  const float rr = (sqrtf(a.hx * a.hx + a.hy * a.hy) + sqrtf(b.hx * b.hx + b.hy * b.hy)) * 1.001f + 1e-3f;
  const float ddx = a.cx - b.cx, ddy = a.cy - b.cy;
  if (ddx * ddx + ddy * ddy > rr * rr) return 0.f;

  const float ox = a.cx, oy = a.cy;
  float2 pa[4], pb[4];
  corners(a, ox, oy, pa);
  corners(b, ox, oy, pb);
  float2 v[kMaxVertices];
  int n = 0;
  float sx = 0.f, sy = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p0 = pa[i], p1 = pa[(i + 1) & 3];
    const float ex = p1.x - p0.x, ey = p1.y - p0.y;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 q0 = pb[j], q1 = pb[(j + 1) & 3];
      const float fx = q1.x - q0.x, fy = q1.y - q0.y;
      const float d0 = cross2(ex, ey, q0.x - p0.x, q0.y - p0.y);   // side of q0, q1 w.r.t. line p
      const float d1 = cross2(ex, ey, q1.x - p0.x, q1.y - p0.y);
      const float e0 = cross2(fx, fy, p0.x - q0.x, p0.y - q0.y);   // side of p0, p1 w.r.t. line q
      const float e1 = cross2(fx, fy, p1.x - q0.x, p1.y - q0.y);
      if (d0 * d1 < 0.f && e0 * e1 < 0.f) {                        // strict on both segments
        const float t = d0 / (d0 - d1);
        const float2 x = make_float2(q0.x + t * fx, q0.y + t * fy);
        if (n < kMaxVertices) {
          v[n++] = x;
          sx += x.x;
          sy += x.y;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (n < kMaxVertices && inside(a, ox, oy, pb[k])) { v[n++] = pb[k]; sx += pb[k].x; sy += pb[k].y; }
    if (n < kMaxVertices && inside(b, ox, oy, pa[k])) { v[n++] = pa[k]; sx += pa[k].x; sy += pa[k].y; }
  }
  if (n < 3) return 0.f;
  const float inv = 1.f / (float)n;
  const float mx = sx * inv, my = sy * inv;
  float key[kMaxVertices];
  for (int k = 0; k < n; ++k) key[k] = pseudo_angle(v[k].x - mx, v[k].y - my);
  for (int k = 1; k < n; ++k) {                    // insertion sort by angle (n <= kMaxVertices)
    const float kk = key[k];
    const float2 vk = v[k];
    int m = k - 1;
    while (m >= 0 && key[m] > kk) { key[m + 1] = key[m]; v[m + 1] = v[m]; --m; }
    key[m + 1] = kk;
    v[m + 1] = vk;
  }
  float area = 0.f;
  for (int k = 1; k + 1 < n; ++k)
    area += cross2(v[k].x - v[0].x, v[k].y - v[0].y, v[k + 1].x - v[0].x, v[k + 1].y - v[0].y);
  return fabsf(area) * 0.5f;
}

}  // namespace
}  // namespace bevb200
