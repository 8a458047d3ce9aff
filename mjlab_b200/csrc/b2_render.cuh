// b2_render.cuh — offscreen frames of the batched scene (the reference's OffscreenRenderer, viewer/offscreen_renderer.py,
// without OpenGL): one ray per pixel against the geoms' poses as the step left them, Lambert shading, one shadow ray.
//
// What is drawn (the items): every static geom once (a geom whose body is welded to the world, drawn from world 0's
// values), then the dynamic geoms of worlds 0 .. noverlay - 1 and of the main world env_idx.  Mesh geoms and geoms
// whose alpha is 0 are not drawn; any other alpha is opaque.  Poses: grid-static geoms from static_pose, height fields
// welded to the world from fixed_pose, every other geom from its world's geom_xpos / geom_xmat.
//
// Launch: a 1-D grid of B2R_TILE x B2R_TILE-pixel tiles, one thread per pixel.  A CTA first culls the items against
// its tile's frustum by bounding sphere (warp ballots and a prefix over the warps build a shared-memory list), then each
// thread casts its pixel's ray against the list and its shadow ray against every item (bounding-sphere reject first).
// A tile whose survivors overflow the list casts against every item.
//
// Conventions (tests/test_render.py reproduces them in fp64): a solid geom is hit where the ray enters it (a ray that
// starts inside sees nothing of it), a plane or height-field surface from either side.  Constants: DESIGN.md §4.
//
// Decoration (the debug visualisers' overlay, tests/test_render_debug_vis.py reproduces it in fp64): a ghost of the
// dynamic geoms at other poses (ghost_xpos / ghost_xmat, sizes of world env_idx, one colour) and arrows (a cylinder
// shaft of radius w and a cone head of base radius 2w and length min(L/2, 4w), apex at `to`).  Decoration items enter
// the tile list after the scene's, so the scene's part of every loop is unchanged.  They are one translucent layer:
// the nearest decoration entry in front of the opaque hit, shaded without shadows, is blended over the opaque colour;
// it casts no shadow and is not in depth or seg.  A frame with decoration is two launches: the scene-only instance of
// the kernel, then the decoration instance, which writes only the pixels decoration covers.
#pragma once
#include "b2_types.h"

#define B2R_TILE 16
#define B2R_LIST 2048  // tile list capacity (items)
#define B2R_INF 3.0e38f
#define B2R_MAXDECOR 64  // arrows per frame
#define B2R_DECOR 12     // floats per arrow record: from[3], to[3], width, rgba[4], padding

// The items' static part, built once per sim (b2_render): static geoms with their pose source, and the dynamic geoms.
struct B2RenderPlan {
  const int* stat;  // [nstat][2] (geom, pose): pose >= 0 row of static_pose, <= -2 row -2 - pose of fixed_pose, -1 world 0
  const int* dyn;   // [ndyn] drawable geoms on bodies that are not welded to the world
  int nstat, ndyn;
};

// One frame's camera and outputs (the host fills it from B2RenderArgs).
struct B2RenderFrame {
  int width, height, ntx;          // image size, tiles per row
  int env_idx, noverlay, nitem;    // main world, overlay worlds 0..noverlay-1, items of the frame
  int track_body;                  // >= 0: the target is subtree_com of this body in world env_idx
  int shadows, brute;
  float lookat[3], distance;
  float fwd[3], right[3], up[3];   // camera axes (z up)
  float tan_y, tan_x;              // tangents of the half field of view
  unsigned char* rgb;
  float* depth;
  int* seg;
  // decoration: items nitem .. nitem + ndeco - 1 of the cull; the first nghost are the ghost of P.dyn, then the arrows
  int ndeco, nghost;
  const float* decor;              // [ndeco - nghost][B2R_DECOR]
  const float* ghost_xpos;         // [ngeom][3]
  const float* ghost_xmat;         // [ngeom][9]
  float ghost_rgba[4];
};

// light: unit direction toward the light; intensity = AMBIENT + DIFFUSE max(0, n.L) (0 when shadowed) + HEAD max(0, -n.d)
#define B2R_LX 0.36f
#define B2R_LY 0.48f
#define B2R_LZ 0.80f
#define B2R_AMBIENT 0.1f
#define B2R_DIFFUSE 0.6f
#define B2R_HEAD 0.3f
#define B2R_CHECKER 0.5f      // checker square of planes (m); odd squares are darkened by B2R_CHECKER_DARK
#define B2R_CHECKER_DARK 0.8f
#define B2R_SHADOW_EPS 1e-3f  // shadow rays start this far off the surface, along its normal
#define B2R_BG_R 153
#define B2R_BG_G 178
#define B2R_BG_B 204

struct B2RItem {
  int world, geom, type;
  const float* pos;  // [3] world position
  const float* mat;  // [9] row-major world rotation (columns: the geom's axes)
};

__device__ __forceinline__ B2RItem b2r_item(const DevModel& m, const DevData& d, const B2RenderPlan& P,
                                            const B2RenderFrame& F, int i) {
  B2RItem it;
  if (i < P.nstat) {
    const int g = P.stat[2 * i], pose = P.stat[2 * i + 1];
    it.world = 0; it.geom = g;
    if (pose >= 0) { it.pos = m.static_pose + 16 * (size_t)pose; it.mat = it.pos + 3; }
    else if (pose <= -2) { it.pos = m.fixed_pose + 16 * (size_t)(-2 - pose); it.mat = it.pos + 3; }
    else { it.pos = d.geom_xpos.p + 3 * g; it.mat = d.geom_xmat.p + 9 * g; }
  } else {
    const int j = i - P.nstat, k = j / P.ndyn, g = P.dyn[j - k * P.ndyn];
    const int w = k < F.noverlay ? k : F.env_idx;
    it.world = w; it.geom = g;
    it.pos = d.geom_xpos.p + (size_t)w * d.geom_xpos.stride + 3 * g;
    it.mat = d.geom_xmat.p + (size_t)w * d.geom_xmat.stride + 9 * g;
  }
  it.type = m.geom_type[it.geom];
  return it;
}

__device__ __forceinline__ const float* b2r_size(const DevModel& m, const B2RItem& it) {
  return m.geom_size.p + (size_t)it.world * m.geom_size.stride + 3 * it.geom;
}
__device__ __forceinline__ const float* b2r_rgba(const DevModel& m, const B2RItem& it) {
  return m.geom_rgba.p + (size_t)it.world * m.geom_rgba.stride + 4 * it.geom;
}

// Bounding sphere about the geom's position: geom_rbound, the rectangle of a finite plane (infinite: B2R_INF), the box
// of a height field's top surface.
__device__ __forceinline__ float b2r_radius(const DevModel& m, const B2RItem& it) {
  const float* s = b2r_size(m, it);
  if (it.type == G_PLANE) return (s[0] > 0.f && s[1] > 0.f) ? sqrtf(s[0] * s[0] + s[1] * s[1]) : B2R_INF;
  if (it.type == G_HFIELD) {
    const float* hs = m.hfield_size + 4 * m.geom_dataid[it.geom];
    return sqrtf(hs[0] * hs[0] + hs[1] * hs[1] + hs[2] * hs[2]);
  }
  return m.geom_rbound.p[(size_t)it.world * m.geom_rbound.stride + it.geom];
}

// Entry interval of the ray o + t d into the slab |x| <= h along one axis: (lo, hi); axis index of the entry face.
__device__ __forceinline__ void b2r_slab(float o, float d, float h, float& lo, float& hi) {
  if (d == 0.f) {
    lo = (fabsf(o) <= h) ? -B2R_INF : B2R_INF;
    hi = (fabsf(o) <= h) ? B2R_INF : -B2R_INF;
    return;
  }
  const float inv = 1.f / d, a = (-h - o) * inv, b = (h - o) * inv;
  lo = fminf(a, b); hi = fmaxf(a, b);
}

// Ray against a z-aligned cylinder of radius r (infinite): entry and exit t, or false.
__device__ __forceinline__ bool b2r_tube(const float* o, const float* d, float r, float& lo, float& hi) {
  const float a = d[0] * d[0] + d[1] * d[1];
  if (a == 0.f) {
    const bool in = o[0] * o[0] + o[1] * o[1] <= r * r;
    lo = in ? -B2R_INF : B2R_INF; hi = in ? B2R_INF : -B2R_INF;
    return in;
  }
  const float tc = -(o[0] * d[0] + o[1] * d[1]) / a, qx = o[0] + tc * d[0], qy = o[1] + tc * d[1];
  const float h = r * r - (qx * qx + qy * qy);
  if (h < 0.f) return false;
  const float dt = sqrtf(h / a);
  lo = tc - dt; hi = tc + dt;
  return true;
}

// Ray against a sphere of radius r at c (local coordinates): entry t, or B2R_INF.
__device__ __forceinline__ float b2r_ball(const float* o, const float* d, float cz, float r) {
  const float oz = o[2] - cz;
  const float a = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  const float tc = -(o[0] * d[0] + o[1] * d[1] + oz * d[2]) / a;
  const float qx = o[0] + tc * d[0], qy = o[1] + tc * d[1], qz = oz + tc * d[2];
  const float h = r * r - (qx * qx + qy * qy + qz * qz);
  return h < 0.f ? B2R_INF : tc - sqrtf(h / a);
}

// Nearest hit of the top surface of a height field (local coordinates, box clipped to (tmin, tmax)): the cells the ray
// crosses, in order, each as its two collision triangles (b2_convex.h: b2c_hfield_tri).
__device__ float b2r_hfield(const DevModel& m, int g, const float* o, const float* d, float tmin, float tmax, float* n) {
  const int id = m.geom_dataid[g], nrow = m.hfield_nrow[id], ncol = m.hfield_ncol[id];
  const float* hs = m.hfield_size + 4 * id;
  const float* z = m.hfield_data + m.hfield_adr[id];
  const float sx = hs[0], sy = hs[1], sz = hs[2];
  float lo, hi, t0 = tmin, t1 = tmax;
  b2r_slab(o[0], d[0], sx, lo, hi); t0 = fmaxf(t0, lo); t1 = fminf(t1, hi);
  b2r_slab(o[1], d[1], sy, lo, hi); t0 = fmaxf(t0, lo); t1 = fminf(t1, hi);
  b2r_slab(o[2] - 0.5f * sz, d[2], 0.5f * sz, lo, hi); t0 = fmaxf(t0, lo); t1 = fminf(t1, hi);
  if (!(t0 <= t1)) return B2R_INF;
  const float dx = 2.f * sx / (float)(ncol - 1), dy = 2.f * sy / (float)(nrow - 1);
  int c = (int)floorf((o[0] + t0 * d[0] + sx) / dx), r = (int)floorf((o[1] + t0 * d[1] + sy) / dy);
  c = min(max(c, 0), ncol - 2); r = min(max(r, 0), nrow - 2);
  const int stx = d[0] > 0.f ? 1 : -1, sty = d[1] > 0.f ? 1 : -1;
  const float idx = d[0] != 0.f ? 1.f / d[0] : B2R_INF, idy = d[1] != 0.f ? 1.f / d[1] : B2R_INF;
  float tx = d[0] != 0.f ? (-sx + (float)(c + (stx > 0)) * dx - o[0]) * idx : B2R_INF;
  float ty = d[1] != 0.f ? (-sy + (float)(r + (sty > 0)) * dy - o[1]) * idy : B2R_INF;
  const float ddx = d[0] != 0.f ? dx * fabsf(idx) : B2R_INF, ddy = d[1] != 0.f ? dy * fabsf(idy) : B2R_INF;
  for (int step = 0; step < nrow + ncol; step++) {
    const float x0 = -sx + dx * (float)c, y0 = -sy + dy * (float)r;
    const float z00 = z[r * ncol + c] * sz, z01 = z[r * ncol + c + 1] * sz;
    const float z10 = z[(r + 1) * ncol + c] * sz, z11 = z[(r + 1) * ncol + c + 1] * sz;
    float best = B2R_INF;
    for (int t = 0; t < 2; t++) {
      // t = 0: (r,c) (r,c+1) (r+1,c+1);  t = 1: (r,c) (r+1,c+1) (r+1,c)
      const float p0[3] = {x0, y0, z00};
      const float p1[3] = {x0 + dx, t ? y0 + dy : y0, t ? z11 : z01};
      const float p2[3] = {t ? x0 : x0 + dx, y0 + dy, t ? z10 : z11};
      const float e1[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
      const float e2[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
      const float pv[3] = {d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0]};
      const float det = e1[0] * pv[0] + e1[1] * pv[1] + e1[2] * pv[2];
      if (det == 0.f) continue;
      const float inv = 1.f / det;
      const float tv[3] = {o[0] - p0[0], o[1] - p0[1], o[2] - p0[2]};
      const float u = (tv[0] * pv[0] + tv[1] * pv[1] + tv[2] * pv[2]) * inv;
      const float qv[3] = {tv[1] * e1[2] - tv[2] * e1[1], tv[2] * e1[0] - tv[0] * e1[2], tv[0] * e1[1] - tv[1] * e1[0]};
      const float v = (d[0] * qv[0] + d[1] * qv[1] + d[2] * qv[2]) * inv;
      const float tt = (e2[0] * qv[0] + e2[1] * qv[1] + e2[2] * qv[2]) * inv;
      const float eps = -1e-5f;  // closes the seams between triangles against fp32 rounding
      if (u < eps || v < eps || u + v > 1.f - eps || !(tt > tmin) || !(tt < best)) continue;
      best = tt;
      n[0] = e1[1] * e2[2] - e1[2] * e2[1]; n[1] = e1[2] * e2[0] - e1[0] * e2[2]; n[2] = e1[0] * e2[1] - e1[1] * e2[0];
    }
    if (best < B2R_INF) return best;
    const float tn = fminf(tx, ty);
    if (tn > t1) break;
    if (tx < ty) { c += stx; tx += ddx; if (c < 0 || c > ncol - 2) break; }
    else { r += sty; ty += ddy; if (r < 0 || r > nrow - 2) break; }
  }
  return B2R_INF;
}

// Nearest entry t in (tmin, tmax) of the ray o + t d (world, d unit) into the item, or B2R_INF; n: world normal there
// (not normalised); *checker: the parity of the plane's checker square (planes only).
__device__ float b2r_hit(const DevModel& m, const B2RItem& it, const float* ow, const float* dw, float tmin, float tmax,
                         float* n, int* checker) {
  const float* R = it.mat;
  const float* s = b2r_size(m, it);
  const float v[3] = {ow[0] - it.pos[0], ow[1] - it.pos[1], ow[2] - it.pos[2]};
  float o[3], d[3], nl[3] = {0.f, 0.f, 0.f};
  for (int k = 0; k < 3; k++) {
    o[k] = R[k] * v[0] + R[3 + k] * v[1] + R[6 + k] * v[2];
    d[k] = R[k] * dw[0] + R[3 + k] * dw[1] + R[6 + k] * dw[2];
  }
  float t = B2R_INF;
  switch (it.type) {
    case G_PLANE: {
      if (d[2] == 0.f) return B2R_INF;
      t = -o[2] / d[2];
      const float x = o[0] + t * d[0], y = o[1] + t * d[1];
      if (s[0] > 0.f && s[1] > 0.f && (fabsf(x) > s[0] || fabsf(y) > s[1])) return B2R_INF;
      nl[2] = 1.f;
      *checker = ((int)floorf(x / B2R_CHECKER) + (int)floorf(y / B2R_CHECKER)) & 1;
      break;
    }
    case G_HFIELD:
      t = b2r_hfield(m, it.geom, o, d, tmin, tmax, nl);
      break;
    case G_SPHERE:
      t = b2r_ball(o, d, 0.f, s[0]);
      for (int k = 0; k < 3; k++) nl[k] = o[k] + t * d[k];
      break;
    case G_ELLIPSOID: {
      const float os[3] = {o[0] / s[0], o[1] / s[1], o[2] / s[2]}, ds[3] = {d[0] / s[0], d[1] / s[1], d[2] / s[2]};
      t = b2r_ball(os, ds, 0.f, 1.f);
      for (int k = 0; k < 3; k++) nl[k] = (o[k] + t * d[k]) / (s[k] * s[k]);
      break;
    }
    case G_CAPSULE: {
      float lo, hi;
      if (b2r_tube(o, d, s[0], lo, hi) && fabsf(o[2] + lo * d[2]) <= s[1]) {
        t = lo;
        nl[0] = o[0] + t * d[0]; nl[1] = o[1] + t * d[1];
      }
      for (int e = -1; e <= 1; e += 2) {
        const float tb = b2r_ball(o, d, e * s[1], s[0]);
        if (tb < t) {
          t = tb;
          nl[0] = o[0] + t * d[0]; nl[1] = o[1] + t * d[1]; nl[2] = o[2] + t * d[2] - e * s[1];
        }
      }
      break;
    }
    case G_CYLINDER: {
      float lo, hi, zl, zh;
      if (!b2r_tube(o, d, s[0], lo, hi)) return B2R_INF;
      b2r_slab(o[2], d[2], s[1], zl, zh);
      if (fmaxf(lo, zl) > fminf(hi, zh)) return B2R_INF;
      if (lo >= zl) { t = lo; nl[0] = o[0] + t * d[0]; nl[1] = o[1] + t * d[1]; }
      else { t = zl; nl[2] = d[2] > 0.f ? -1.f : 1.f; }
      break;
    }
    case G_BOX: {
      float lo = -B2R_INF, hi = B2R_INF;
      int ax = 0;
      for (int k = 0; k < 3; k++) {
        float a, b;
        b2r_slab(o[k], d[k], s[k], a, b);
        if (a > lo) { lo = a; ax = k; }
        hi = fminf(hi, b);
      }
      if (lo > hi) return B2R_INF;
      t = lo;
      nl[ax] = d[ax] > 0.f ? -1.f : 1.f;
      break;
    }
    default:
      return B2R_INF;
  }
  if (!(t > tmin) || !(t < tmax)) return B2R_INF;
  for (int k = 0; k < 3; k++) n[k] = R[3 * k] * nl[0] + R[3 * k + 1] * nl[1] + R[3 * k + 2] * nl[2];
  return t;
}

// false when the ray o + t d, t in (0, tmax), certainly misses the sphere (c, r).
__device__ __forceinline__ bool b2r_near(const float* o, const float* d, const float* c, float r, float tmax) {
  if (r >= B2R_INF) return true;
  const float v[3] = {c[0] - o[0], c[1] - o[1], c[2] - o[2]};
  const float b = v[0] * d[0] + v[1] * d[1] + v[2] * d[2];
  const float rr = r * 1.001f + 1e-4f;
  if (b < -rr || b - rr > tmax) return false;
  const float q[3] = {v[0] - b * d[0], v[1] - b * d[1], v[2] - b * d[2]};
  return q[0] * q[0] + q[1] * q[1] + q[2] * q[2] <= rr * rr;
}

__device__ __forceinline__ bool b2r_drawn(const DevModel& m, const B2RItem& it) { return b2r_rgba(m, it)[3] != 0.f; }

// Direction (unnormalised) of the ray through image point (x, y) in pixels from the top-left corner.
__device__ __forceinline__ void b2r_dir(const B2RenderFrame& F, float x, float y, float* dir) {
  const float a = (2.f * x / (float)F.width - 1.f) * F.tan_x, b = (1.f - 2.f * y / (float)F.height) * F.tan_y;
  for (int k = 0; k < 3; k++) dir[k] = F.fwd[k] + a * F.right[k] + b * F.up[k];
}

// ---- decoration items

// Ghost item j < F.nghost: the dynamic geom P.dyn[j] at the ghost's pose, with world env_idx's size and bound.
__device__ __forceinline__ B2RItem b2r_ghost(const DevModel& m, const B2RenderPlan& P, const B2RenderFrame& F, int j) {
  B2RItem it;
  it.world = F.env_idx; it.geom = P.dyn[j];
  it.pos = F.ghost_xpos + 3 * it.geom; it.mat = F.ghost_xmat + 9 * it.geom;
  it.type = m.geom_type[it.geom];
  return it;
}

// An arrow record's unit axis, length L and head length h; false when it is not drawn (L < 1e-6 or alpha 0).
__device__ __forceinline__ bool b2r_arrow_axis(const float* a, float* ax, float& L, float& h) {
  for (int k = 0; k < 3; k++) ax[k] = a[3 + k] - a[k];
  L = sqrtf(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
  if (!(L >= 1e-6f) || a[10] == 0.f) return false;
  const float inv = 1.f / L;
  for (int k = 0; k < 3; k++) ax[k] *= inv;
  h = fminf(0.5f * L, 4.f * a[6]);
  return true;
}

// Bounding sphere (c, r) of decoration item j; false when the item is not drawn.
__device__ __forceinline__ bool b2r_deco_bound(const DevModel& m, const B2RenderPlan& P, const B2RenderFrame& F, int j,
                                               float* c, float& r) {
  if (j < F.nghost) {
    const B2RItem it = b2r_ghost(m, P, F, j);
    for (int k = 0; k < 3; k++) c[k] = it.pos[k];
    r = b2r_radius(m, it);
    return true;
  }
  const float* a = F.decor + B2R_DECOR * (j - F.nghost);
  float ax[3], L, h;
  if (!b2r_arrow_axis(a, ax, L, h)) return false;
  for (int k = 0; k < 3; k++) c[k] = 0.5f * (a[k] + a[3 + k]);
  r = sqrtf(0.25f * L * L + 4.f * a[6] * a[6]);
  return true;
}

// Entry t in (0, tmax) of the ray ow + t dw (d unit) into the arrow record a, or B2R_INF; n: world normal there (not
// normalised).  In the arrow's frame (z along the axis, `from` at the origin) the shaft is |xy| <= w, 0 <= z <= L - h,
// and the head is the solid cone of apex (0, 0, L) and base radius 2w at z = L - h.
__device__ float b2r_arrow(const float* a, const float* ow, const float* dw, float tmax, float* n) {
  float ez[3], L, h;
  if (!b2r_arrow_axis(a, ez, L, h)) return B2R_INF;
  const float w = a[6];
  float ex[3], ey[3];
  {
    const float hx = fabsf(ez[0]) < 0.9f ? 1.f : 0.f, hy = 1.f - hx, p = hx * ez[0] + hy * ez[1];
    ex[0] = hx - p * ez[0]; ex[1] = hy - p * ez[1]; ex[2] = -p * ez[2];
    const float inv = rsqrtf(ex[0] * ex[0] + ex[1] * ex[1] + ex[2] * ex[2]);
    for (int k = 0; k < 3; k++) ex[k] *= inv;
    ey[0] = ez[1] * ex[2] - ez[2] * ex[1]; ey[1] = ez[2] * ex[0] - ez[0] * ex[2]; ey[2] = ez[0] * ex[1] - ez[1] * ex[0];
  }
  const float v[3] = {ow[0] - a[0], ow[1] - a[1], ow[2] - a[2]};
  const float o[3] = {ex[0] * v[0] + ex[1] * v[1] + ex[2] * v[2], ey[0] * v[0] + ey[1] * v[1] + ey[2] * v[2],
                      ez[0] * v[0] + ez[1] * v[1] + ez[2] * v[2]};
  const float d[3] = {ex[0] * dw[0] + ex[1] * dw[1] + ex[2] * dw[2], ey[0] * dw[0] + ey[1] * dw[1] + ey[2] * dw[2],
                      ez[0] * dw[0] + ez[1] * dw[1] + ez[2] * dw[2]};
  float t = B2R_INF, nl[3] = {0.f, 0.f, 0.f}, lo, hi, zl, zh;
  // shaft: a cylinder with flat caps
  if (b2r_tube(o, d, w, lo, hi)) {
    b2r_slab(o[2] - 0.5f * (L - h), d[2], 0.5f * (L - h), zl, zh);
    const float e = fmaxf(lo, zl);
    if (e <= fminf(hi, zh) && e > 0.f) {
      t = e;
      if (lo >= zl) { nl[0] = o[0] + t * d[0]; nl[1] = o[1] + t * d[1]; }
      else nl[2] = d[2] > 0.f ? -1.f : 1.f;
    }
  }
  // head: the ray's interval (lo, hi) in the cone's nappe z <= L, clipped to L - h <= z <= L
  {
    const float k2 = (2.f * w / h) * (2.f * w / h), qz = o[2] - L;
    const float A = d[0] * d[0] + d[1] * d[1] - k2 * d[2] * d[2];
    const float B = o[0] * d[0] + o[1] * d[1] - k2 * qz * d[2];
    const float C = o[0] * o[0] + o[1] * o[1] - k2 * qz * qz;
    const float disc = B * B - A * C;
    float r1 = B2R_INF, r2 = B2R_INF;
    bool v1 = false, v2 = false;
    if (A != 0.f && disc >= 0.f) {
      const float sq = sqrtf(disc), x1 = (-B - sq) / A, x2 = (-B + sq) / A;
      r1 = fminf(x1, x2); r2 = fmaxf(x1, x2);
      v1 = qz + r1 * d[2] <= 0.f; v2 = qz + r2 * d[2] <= 0.f;
    } else if (A == 0.f && B != 0.f) {
      r1 = -0.5f * C / B;
      v1 = qz + r1 * d[2] <= 0.f;
    }
    lo = B2R_INF; hi = -B2R_INF;
    if (v1 && v2) { lo = r1; hi = r2; }
    else if (v1 || v2) {  // the ray leaves the nappe toward +z, or enters it toward -z and stays
      const float r = v1 ? r1 : r2;
      if (d[2] < 0.f) { lo = r; hi = B2R_INF; }
      else { lo = -B2R_INF; hi = r; }
    }
    b2r_slab(o[2] - (L - 0.5f * h), d[2], 0.5f * h, zl, zh);
    const float e = fmaxf(lo, zl);
    if (e <= fminf(hi, zh) && e > 0.f && e < t) {
      t = e;
      if (lo >= zl) { nl[0] = o[0] + t * d[0]; nl[1] = o[1] + t * d[1]; nl[2] = -k2 * (qz + t * d[2]); }
      else { nl[0] = 0.f; nl[1] = 0.f; nl[2] = d[2] > 0.f ? -1.f : 1.f; }
    }
  }
  if (!(t < tmax)) return B2R_INF;
  for (int k = 0; k < 3; k++) n[k] = ex[k] * nl[0] + ey[k] * nl[1] + ez[k] * nl[2];
  return t;
}

// The decoration pass of one ray o + t dir (dir unit): the nearest decoration item among entries first .. last - 1 of
// the tile list (all: every item) entered before `best`, or -1; dc: its shaded, clamped colour and its alpha.  The
// decoration instance of b2_render_kernel.
__device__ __forceinline__ int b2r_decorate(const DevModel& m, const B2RenderPlan& P, const B2RenderFrame& F,
                                         const int* list, int first, int last, bool all, const float* o,
                                         const float* dir, float best, float* dc) {
  int deco = -1;
  float dbest = best, dn[3];
  for (int j = first; j < last; j++) {
    const int k = all ? j : list[j] - F.nitem;
    float nn[3], t;
    if (k < F.nghost) {
      const B2RItem it = b2r_ghost(m, P, F, k);
      if (!b2r_near(o, dir, it.pos, b2r_radius(m, it), dbest)) continue;
      int ck;
      t = b2r_hit(m, it, o, dir, 0.f, dbest, nn, &ck);
    } else {
      t = b2r_arrow(F.decor + B2R_DECOR * (k - F.nghost), o, dir, dbest, nn);
    }
    if (t < dbest) { dbest = t; deco = k; dn[0] = nn[0]; dn[1] = nn[1]; dn[2] = nn[2]; }
  }
  if (deco >= 0) {
    const float inv = rsqrtf(dn[0] * dn[0] + dn[1] * dn[1] + dn[2] * dn[2]);
    const float sg = (dn[0] * dir[0] + dn[1] * dir[1] + dn[2] * dir[2]) > 0.f ? -inv : inv;
    for (int k = 0; k < 3; k++) dn[k] *= sg;
    const float light = B2R_AMBIENT + B2R_DIFFUSE * fmaxf(0.f, dn[0] * B2R_LX + dn[1] * B2R_LY + dn[2] * B2R_LZ) +
                        B2R_HEAD * fmaxf(0.f, -(dn[0] * dir[0] + dn[1] * dir[1] + dn[2] * dir[2]));
    const float* c = deco < F.nghost ? F.ghost_rgba : F.decor + B2R_DECOR * (deco - F.nghost) + 7;
    for (int k = 0; k < 3; k++) dc[k] = fminf(fmaxf(c[k] * light, 0.f), 1.f);
    dc[3] = c[3];
  }
  return deco;
}

// DECO = false draws the scene: every pixel's rgb, depth and seg.  DECO = true runs after it on frames with decoration
// and writes only the rgb of the pixels a decoration item covers, blended over the scene's colour, which it recomputes
// for them.  So the scene's outputs come from the same instance with decoration or without, bit for bit (two
// instances of the scene's code need not round alike: the compiler contracts their arithmetic independently), and
// the scene-only instance keeps its register budget.
template <bool DECO>
__global__ void __launch_bounds__(B2R_TILE * B2R_TILE) b2_render_kernel(DevModel m, DevData d, B2RenderPlan P,
                                                                        B2RenderFrame F) {
  __shared__ int list[B2R_LIST];
  __shared__ int warp_n[B2R_TILE * B2R_TILE / 32], warp_s[B2R_TILE * B2R_TILE / 32];
  __shared__ int nlist, nscene, overflow;  // nscene: the list's scene items, before its decoration items
  __shared__ float eye[3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile_x = blockIdx.x % F.ntx, tile_y = blockIdx.x / F.ntx;
  const int px = tile_x * B2R_TILE + tid % B2R_TILE, py = tile_y * B2R_TILE + tid / B2R_TILE;
  if (tid == 0) {
    const float* c = F.lookat;
    if (F.track_body >= 0) c = d.subtree_com.p + (size_t)F.env_idx * d.subtree_com.stride + 3 * F.track_body;
    for (int k = 0; k < 3; k++) eye[k] = c[k] - F.distance * F.fwd[k];
    nlist = nscene = 0;
    overflow = F.brute;
  }
  __syncthreads();
  const float o[3] = {eye[0], eye[1], eye[2]};
  // ---- tile cull: the four side planes of the tile's frustum (through the eye) and the camera's front half-space
  if (!F.brute) {
    float pl[4][3];
    {
      const float x0 = (float)(tile_x * B2R_TILE), x1 = fminf(x0 + B2R_TILE, (float)F.width);
      const float y0 = (float)(tile_y * B2R_TILE), y1 = fminf(y0 + B2R_TILE, (float)F.height);
      float c[4][3], mid[3];
      b2r_dir(F, x0, y0, c[0]); b2r_dir(F, x1, y0, c[1]); b2r_dir(F, x1, y1, c[2]); b2r_dir(F, x0, y1, c[3]);
      b2r_dir(F, 0.5f * (x0 + x1), 0.5f * (y0 + y1), mid);
      for (int e = 0; e < 4; e++) {
        const float* a = c[e];
        const float* b = c[(e + 1) & 3];
        float nx = a[1] * b[2] - a[2] * b[1], ny = a[2] * b[0] - a[0] * b[2], nz = a[0] * b[1] - a[1] * b[0];
        const float inv = rsqrtf(nx * nx + ny * ny + nz * nz) * (nx * mid[0] + ny * mid[1] + nz * mid[2] < 0.f ? -1.f : 1.f);
        pl[e][0] = nx * inv; pl[e][1] = ny * inv; pl[e][2] = nz * inv;
      }
    }
    // the scene's items 0 .. nitem - 1, then the decoration's nitem .. nitem + ndeco - 1 (list entry nitem + j)
    const int ncull = DECO ? F.nitem + F.ndeco : F.nitem;
    for (int base = 0; base < ncull; base += B2R_TILE * B2R_TILE) {
      const int i = base + tid;
      bool keep = false;
      float c[3], r = 0.f;
      if (i < F.nitem) {
        const B2RItem it = b2r_item(m, d, P, F, i);
        keep = b2r_drawn(m, it);
        if (keep) { r = b2r_radius(m, it); c[0] = it.pos[0]; c[1] = it.pos[1]; c[2] = it.pos[2]; }
      } else if (DECO && i < ncull) {
        keep = b2r_deco_bound(m, P, F, i - F.nitem, c, r);
      }
      if (keep && r < B2R_INF) {
        const float v[3] = {c[0] - o[0], c[1] - o[1], c[2] - o[2]};
        const float rr = r * 1.001f + 1e-4f * (1.f + sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
        keep = v[0] * F.fwd[0] + v[1] * F.fwd[1] + v[2] * F.fwd[2] >= -rr;
        for (int e = 0; e < 4; e++) keep &= pl[e][0] * v[0] + pl[e][1] * v[1] + pl[e][2] * v[2] >= -rr;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      const unsigned bal_scene = DECO ? __ballot_sync(0xffffffffu, keep && i < F.nitem) : bal;
      if (lane == 0) { warp_n[warp] = __popc(bal); warp_s[warp] = __popc(bal_scene); }
      __syncthreads();
      int off = nlist;
      for (int w = 0; w < warp; w++) off += warp_n[w];
      off += __popc(bal & ((1u << lane) - 1u));
      if (keep) {
        if (off < B2R_LIST) list[off] = i;
        else overflow = 1;
      }
      __syncthreads();
      if (tid == 0)
        for (int w = 0; w < B2R_TILE * B2R_TILE / 32; w++) { nlist += warp_n[w]; nscene += warp_s[w]; }
      __syncthreads();
    }
  }
  if (px >= F.width || py >= F.height) return;
  // ---- primary ray
  float dir[3];
  b2r_dir(F, (float)px + 0.5f, (float)py + 0.5f, dir);
  {
    const float inv = rsqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    for (int k = 0; k < 3; k++) dir[k] *= inv;
  }
  const bool all = overflow != 0;
  const int count = all ? F.nitem : nscene;
  float best = B2R_INF, n[3] = {0.f, 0.f, 1.f};
  int hit = -1, checker = 0;
  for (int j = 0; j < count; j++) {
    const int i = all ? j : list[j];
    const B2RItem it = b2r_item(m, d, P, F, i);
    if (all && !b2r_drawn(m, it)) continue;
    if (!b2r_near(o, dir, it.pos, b2r_radius(m, it), best)) continue;
    float nn[3];
    int ck = 0;
    const float t = b2r_hit(m, it, o, dir, 0.f, best, nn, &ck);
    if (t < best) { best = t; hit = i; checker = ck; n[0] = nn[0]; n[1] = nn[1]; n[2] = nn[2]; }
  }
  const float L[3] = {B2R_LX, B2R_LY, B2R_LZ};
  // ---- decoration: the nearest item entered before the opaque hit, shaded without shadows (dc: colour and alpha)
  int deco = -1;
  float dc[4];
  if (DECO) {
    deco = b2r_decorate(m, P, F, list, all ? 0 : nscene, all ? F.ndeco : nlist, all, o, dir, best, dc);
    if (deco < 0) return;  // the scene instance drew this pixel
  }
  const size_t pix = (size_t)py * F.width + px;
  if (hit < 0) {
    if (!DECO) {
      F.rgb[3 * pix] = B2R_BG_R; F.rgb[3 * pix + 1] = B2R_BG_G; F.rgb[3 * pix + 2] = B2R_BG_B;
      if (F.depth) F.depth[pix] = __int_as_float(0x7f800000);
      if (F.seg) { F.seg[2 * pix] = -1; F.seg[2 * pix + 1] = -1; }
    } else {
      const float bg[3] = {B2R_BG_R / 255.f, B2R_BG_G / 255.f, B2R_BG_B / 255.f};
      for (int k = 0; k < 3; k++)
        F.rgb[3 * pix + k] = (unsigned char)((dc[3] * dc[k] + (1.f - dc[3]) * bg[k]) * 255.f + 0.5f);
    }
    return;
  }
  const B2RItem hi = b2r_item(m, d, P, F, hit);
  {
    const float inv = rsqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    const float sg = (n[0] * dir[0] + n[1] * dir[1] + n[2] * dir[2]) > 0.f ? -inv : inv;  // toward the camera
    for (int k = 0; k < 3; k++) n[k] *= sg;
  }
  float diff = fmaxf(0.f, n[0] * L[0] + n[1] * L[1] + n[2] * L[2]);
  if (F.shadows && diff > 0.f) {
    // ---- shadow ray toward the light, against every scene item
    float p[3];
    for (int k = 0; k < 3; k++) p[k] = o[k] + best * dir[k] + B2R_SHADOW_EPS * n[k];
    for (int i = 0; i < F.nitem && diff > 0.f; i++) {
      const B2RItem it = b2r_item(m, d, P, F, i);
      if (!b2r_drawn(m, it) || !b2r_near(p, L, it.pos, b2r_radius(m, it), B2R_INF)) continue;
      float nn[3];
      int ck;
      if (b2r_hit(m, it, p, L, 0.f, B2R_INF, nn, &ck) < B2R_INF) diff = 0.f;
    }
  }
  const float head = fmaxf(0.f, -(n[0] * dir[0] + n[1] * dir[1] + n[2] * dir[2]));
  float light = B2R_AMBIENT + B2R_DIFFUSE * diff + B2R_HEAD * head;
  if (hi.type == G_PLANE && checker) light *= B2R_CHECKER_DARK;
  const float* rgba = b2r_rgba(m, hi);
  if (!DECO) {
    for (int k = 0; k < 3; k++) F.rgb[3 * pix + k] = (unsigned char)(fminf(fmaxf(rgba[k] * light, 0.f), 1.f) * 255.f + 0.5f);
    if (F.depth) F.depth[pix] = best * (dir[0] * F.fwd[0] + dir[1] * F.fwd[1] + dir[2] * F.fwd[2]);
    if (F.seg) { F.seg[2 * pix] = hi.world; F.seg[2 * pix + 1] = hi.geom; }
  } else {
    for (int k = 0; k < 3; k++) {
      const float co = fminf(fmaxf(rgba[k] * light, 0.f), 1.f);
      F.rgb[3 * pix + k] = (unsigned char)((dc[3] * dc[k] + (1.f - dc[3]) * co) * 255.f + 0.5f);
    }
  }
}
