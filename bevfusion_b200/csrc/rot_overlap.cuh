// The rotated BEV overlap of two boxes, shared by the NMS / IoU kernels (box_nms.cu) and the TransFusion
// assignment cost (transfusion_assign.cu).  Internal header.
//
// Boxes are [x1, y1, x2, y2, ry] fp32.  A box is the axis-aligned extent turned by ry about its centre:
//   x' = (x - cx) cos r + (y - cy) sin r + cx,   y' = -(x - cx) sin r + (y - cy) cos r + cy.
// The overlap is the area of box a clipped by box b (Sutherland-Hodgman): a's corners are taken into b's own frame,
// where b is [-hx, hx] x [-hy, hy], cut by b's four sides in turn (a vertex on a side is kept, a cut lands exactly
// on the side), and summed as a triangle fan.  Nothing tests one edge against another, so collinear or
// touching edges (abutting or nested boxes, yaw + pi, a square turned by pi / 2) cannot add a vertex off the true
// polygon: a rounding error moves a vertex by about the rounding of the coordinates, and the area by as little.
#pragma once
#include "common.cuh"

namespace bevb200 {
namespace {

// Vertex buffer of the clipped polygon: a quadrilateral cut by four lines has at most 8 vertices.  The pushes are
// guarded anyway, so rounding in a near-degenerate pair can never write past the buffer.
constexpr int kMaxVertices = 12;

struct RotBox {
  float x1, y1, hx, hy, c, s;   // low corner, half extents, cos / sin of ry
};

__device__ __forceinline__ RotBox load_rot(const float *b) {
  RotBox r;
  r.x1 = b[0];
  r.y1 = b[1];
  r.hx = (b[2] - b[0]) * 0.5f;
  r.hy = (b[3] - b[1]) * 0.5f;
  sincosf(b[4], &r.s, &r.c);
  return r;
}

__device__ __forceinline__ float cross2(float ax, float ay, float bx, float by) { return ax * by - ay * bx; }

// Keeps the part of the polygon p[0, n) with sign * coordinate kAxis <= lim in q; returns its vertex count.  A
// vertex with a NaN coordinate is dropped and starts no cut.
template <int kAxis>
__device__ __forceinline__ int clip_side(const float2 *p, int n, float sign, float lim, float2 *q) {
  int m = 0;
  for (int i = 0; i < n; ++i) {
    const float2 u = p[i], w = p[i + 1 < n ? i + 1 : 0];
    const float du = lim - sign * (kAxis ? u.y : u.x), dw = lim - sign * (kAxis ? w.y : w.x);
    if (du >= 0.f && m < kMaxVertices) q[m++] = u;
    if (((du >= 0.f && dw < 0.f) || (du < 0.f && dw >= 0.f)) && m < kMaxVertices) {
      const float t = du / (du - dw);
      q[m++] = kAxis ? make_float2(u.x + t * (w.x - u.x), sign * lim) : make_float2(sign * lim, u.y + t * (w.y - u.y));
    }
  }
  return m;
}

__device__ __forceinline__ float rot_overlap(const RotBox &a, const RotBox &b) {
  // a's centre relative to b's, from the corners: (x1a - x1b) is exact for nearby boxes, where rounded centres
  // would carry the rounding of positions up to 61 m (the CenterHead range) into the polygon.
  const float ox = (a.x1 - b.x1) + (a.hx - b.hx), oy = (a.y1 - b.y1) + (a.hy - b.hy);
  // Conservative early-out: circumscribed circles apart by a relative 1e-3 plus 1e-3 overlap nowhere.  NaN
  // compares false and takes the full path, which gives 0.
  const float rr = (sqrtf(a.hx * a.hx + a.hy * a.hy) + sqrtf(b.hx * b.hx + b.hy * b.hy)) * 1.001f + 1e-3f;
  if (ox * ox + oy * oy > rr * rr) return 0.f;

  // In b's frame (turned back by -rb): a's centre, and a's axes turned by ra - rb.
  const float lx = ox * b.c - oy * b.s, ly = ox * b.s + oy * b.c;
  const float c = a.c * b.c + a.s * b.s, s = a.s * b.c - a.c * b.s;
  float2 p[kMaxVertices], q[kMaxVertices];
  const float xs[4] = {-a.hx, a.hx, a.hx, -a.hx}, ys[4] = {-a.hy, -a.hy, a.hy, a.hy};
#pragma unroll
  for (int k = 0; k < 4; ++k) p[k] = make_float2(xs[k] * c + ys[k] * s + lx, -xs[k] * s + ys[k] * c + ly);
  int n = clip_side<0>(p, 4, 1.f, b.hx, q);
  n = clip_side<0>(q, n, -1.f, b.hx, p);
  n = clip_side<1>(p, n, 1.f, b.hy, q);
  n = clip_side<1>(q, n, -1.f, b.hy, p);
  if (n < 3) return 0.f;
  float area = 0.f;
  for (int k = 1; k + 1 < n; ++k)
    area += cross2(p[k].x - p[0].x, p[k].y - p[0].y, p[k + 1].x - p[0].x, p[k + 1].y - p[0].y);
  return fabsf(area) * 0.5f;
}

}  // namespace
}  // namespace bevb200
