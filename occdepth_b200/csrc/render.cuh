// Camera views of a class map: the per-ray voxel walk of occd_render_classes (include/occdepth_b200.h, "Camera
// views").  Camera: M (3x3) = R^-1 K^-1 and o = -R^-1 t for E = [R | t] grid frame -> camera frame (R^T for a rigid
// E), o the camera centre in the grid frame.  For pixel (u, v), in float64 without FMA contraction:
//   d_r   = ((M[r][0] * u + M[r][1] * v) + M[r][2])                 the ray o + t d; t is the camera-frame z
//   t_a(i) = ((origin_a + i * voxel) - o_a) * r_a,  r_a = 1 / d_a    boundary i of axis a, from the integer index
// Slab: an axis with d_a == 0 is never stepped and keeps the ray only if origin_a <= o_a < origin_a + G_a * voxel;
// [t_lo, t_hi] = the intersection of [min, max](t_a(0), t_a(G_a)) over the other axes.  t0 = max(t_lo, near), t_end =
// min(t_hi, far); t0 >= t_end is a miss.  First voxel: floor((o + t0 * d - origin) / voxel), clamped into [0, G_a - 1].
// Walk: test the voxel (a hit is empty != c != ignore); step the axis whose next boundary time is least (ties: x,
// then y, then z); stop with a miss when that time is >= t_end, the index leaves the grid, or after G_x + G_y + G_z + 3
// voxels.  A voxel's entry time is t0 for the first, max(previous entry, the crossed boundary's time) after it.
// Every min / max is a plain comparison (a > b ? a : b), so signed zeros pick the same operand everywhere.  Each step
// is one correctly rounded IEEE operation, so the device, the host build in tests/host_emul/ and numpy's element-wise
// float64 restatement give the same bits.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_fp16.h>
#include "scene_map.cuh"      // mul_rn, add_rn, sub_rn, div_rn and their float32 twins

namespace rnd {

#define RND_HD __host__ __device__ __forceinline__

struct Camera {
  double M[9];                // row-major R^-1 K^-1
  double o[3];                // the camera centre in the grid frame
};

struct Grid {
  double origin[3], voxel;    // the grid's corner and edge
  int G[3];                   // dims along x, y, z
  long long s[3];             // element strides of x, y, z inside one map
  int empty, ignore;          // the classes a ray passes through
  double near_t, far_t;       // the ray interval, near >= 0, far > near (far may be +inf)
};

struct Hit {
  long long off;              // the hit voxel's element offset, -1 on a miss
  double t;                   // its entry time (+inf on a miss)
  int cls;                    // its class (the grid's empty on a miss)
};

RND_HD double lt_min(double a, double b) { return a < b ? a : b; }
RND_HD double gt_max(double a, double b) { return a > b ? a : b; }

// position of boundary i of axis a, and its time along the ray
RND_HD double boundary_time(const Grid& g, const double* o, const double* r, int a, int i) {
  return smap::mul_rn(smap::sub_rn(smap::add_rn(g.origin[a], smap::mul_rn((double)i, g.voxel)), o[a]), r[a]);
}

template <typename T>
RND_HD T ld(const T* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// Every voxel of pixel (u, v)'s ray, in order: visit(off, t) with the voxel's element offset (offsets g.s) and entry
// time, returning true to stop the walk there.  The one walk both renders take; returns whether a visit stopped it.
template <typename Visit>
RND_HD bool walk_ray(const Camera& c, const Grid& g, int u, int v, Visit&& visit) {
  using namespace smap;
  const double uu = (double)u, vv = (double)v;
  double d[3], r[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    d[a] = add_rn(add_rn(mul_rn(c.M[3 * a], uu), mul_rn(c.M[3 * a + 1], vv)), c.M[3 * a + 2]);
  double t_lo = -INFINITY, t_hi = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (d[a] == 0.0) {
      r[a] = 0.0;
      const double hi = add_rn(g.origin[a], mul_rn((double)g.G[a], g.voxel));
      if (!(g.origin[a] <= c.o[a] && c.o[a] < hi)) return false;
    } else {
      r[a] = div_rn(1.0, d[a]);
      const double ta = boundary_time(g, c.o, r, a, 0), tb = boundary_time(g, c.o, r, a, g.G[a]);
      t_lo = gt_max(t_lo, lt_min(ta, tb));
      t_hi = lt_min(t_hi, gt_max(ta, tb));
    }
  }
  const double t0 = gt_max(t_lo, g.near_t), t_end = lt_min(t_hi, g.far_t);
  if (!(t0 < t_end)) return false;
  int idx[3], step[3];
  double tn[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double f = floor(div_rn(sub_rn(add_rn(c.o[a], mul_rn(t0, d[a])), g.origin[a]), g.voxel));
    f = f < 0.0 ? 0.0 : f;
    f = f > (double)(g.G[a] - 1) ? (double)(g.G[a] - 1) : f;
    idx[a] = (int)f;
    step[a] = d[a] > 0.0 ? 1 : -1;
    tn[a] = d[a] == 0.0 ? INFINITY : boundary_time(g, c.o, r, a, idx[a] + (d[a] > 0.0 ? 1 : 0));
  }
  double t = t0;
  const int cap = g.G[0] + g.G[1] + g.G[2] + 3;
  for (int n = 0; n < cap; ++n) {
    const long long off = (long long)idx[0] * g.s[0] + (long long)idx[1] * g.s[1] + (long long)idx[2] * g.s[2];
    if (visit(off, t)) return true;
    // the axis with the least next boundary time, x before y before z on ties; every array index below is a
    // constant, so the walk's state stays in registers
    const int a = tn[1] < tn[0] ? (tn[2] < tn[1] ? 2 : 1) : (tn[2] < tn[0] ? 2 : 0);
    const double tm = a == 0 ? tn[0] : (a == 1 ? tn[1] : tn[2]);
    if (!(tm < t_end)) return false;
    t = gt_max(t, tm);
    bool in = true;
#pragma unroll
    for (int b = 0; b < 3; ++b)
      if (a == b) {
        idx[b] += step[b];
        in = idx[b] >= 0 && idx[b] < g.G[b];
        tn[b] = boundary_time(g, c.o, r, b, idx[b] + (step[b] > 0 ? 1 : 0));
      }
    if (!in) return false;
  }
  return false;
}

// The first visible voxel along pixel (u, v)'s ray through `map` (one item's map, offsets g.s)
RND_HD Hit cast_ray(const Camera& c, const Grid& g, const uint16_t* map, int u, int v) {
  Hit h;
  const bool hit = walk_ray(c, g, u, v, [&](long long off, double t) {
    const int cls = ld(map + off);
    if (cls == g.empty || cls == g.ignore) return false;
    h.off = off;
    h.t = t;
    h.cls = cls;
    return true;
  });
  // the miss is written after the walk, not before it: set first, it would hold registers through the whole loop
  if (!hit) {
    h.off = -1;
    h.t = INFINITY;
    h.cls = g.empty;
  }
  return h;
}

// ---- soft views: each ray's float16 class probabilities composited front to back (occd_render_probs) -------------
// A voxel is occupied with probability 1 - p(empty) and then has class c with weight p(c).  Over the voxels of the
// walk above (g.empty is the empty channel), in float32 with one correctly rounded operation per step, from T = 1,
// D = -0 and S[c] = 0:
//   skip the voxel if class_map is given and holds g.ignore there, or if e = p[empty] == 1 (no other channel read);
//   S[c] += T * p[c] for c != empty;  Tn = T * e, w = T - Tn, D += w * (float)t, T = Tn;  stop once T <= t_min.
// Pixel: opacity = 1 - T, depth = D / opacity (+inf when opacity <= 0), channel empty = T and channel c = S[c]; the
// class is the first maximum over the channels (strict >, from channel 0), then lut[class] when a lut is given.
// Probabilities are not clamped; NaN propagates.
struct SoftIn {
  const __half* probs;        // one item's [C][plane], planes cstride elements apart
  long long cstride;
  const uint16_t* cmap;       // one item's class map, or NULL
  int C;
  float t_min;                // in [0, 1)
  const uint16_t* lut;        // C remapped class ids, or NULL
};

// Pixel (u, v)'s soft view: the class, depth, opacity and C float16 channels (at probs[c * pstride]); an output
// that is NULL is not written
template <int CMAX>
RND_HD void composite_ray(const Camera& c, const Grid& g, const SoftIn& in, int u, int v, uint16_t* cls,
                          float* depth, float* opacity, __half* probs, long long pstride) {
  using namespace smap;
  float S[CMAX];
#pragma unroll
  for (int k = 0; k < CMAX; ++k) S[k] = 0.f;
  float T = 1.f, D = -0.f;    // -0 is IEEE addition's identity: D is exactly its first term, a -0 entry time kept
  walk_ray(c, g, u, v, [&](long long off, double t) {
    if (in.cmap && (int)ld(in.cmap + off) == g.ignore) return false;
    const float e = __half2float(ld(in.probs + g.empty * in.cstride + off));
    if (e == 1.f) return false;
    // every channel's load in flight before the first use; two channels per register
    __half2 p[CMAX / 2];
#pragma unroll
    for (int k = 0; k < CMAX; k += 2) {
      const __half lo = k < in.C && k != g.empty ? ld(in.probs + k * in.cstride + off) : __float2half(0.f);
      const __half hi = k + 1 < in.C && k + 1 != g.empty ? ld(in.probs + (k + 1) * in.cstride + off)
                                                          : __float2half(0.f);
      p[k / 2] = __halves2half2(lo, hi);
    }
#pragma unroll
    for (int k = 0; k < CMAX; ++k)
      if (k < in.C && k != g.empty) {
        const float pk = (k & 1) ? __high2float(p[k / 2]) : __low2float(p[k / 2]);
        S[k] = fadd_rn(S[k], fmul_rn(T, pk));
      }
    const float Tn = fmul_rn(T, e);
    D = fadd_rn(D, fmul_rn(fsub_rn(T, Tn), (float)t));
    T = Tn;
    return T <= in.t_min;
  });
  const float o = fsub_rn(1.f, T);
  if (opacity) *opacity = o;
  if (depth) *depth = o > 0.f ? fdiv_rn(D, o) : INFINITY;
  float best = 0.f;
  int arg = 0;
#pragma unroll
  for (int k = 0; k < CMAX; ++k)
    if (k < in.C) {
      const float x = k == g.empty ? T : S[k];
      if (probs) probs[k * pstride] = __float2half_rn(x);
      if (k == 0 || x > best) {
        best = x;
        arg = k;
      }
    }
  if (cls) *cls = in.lut ? in.lut[arg] : (uint16_t)arg;
}

}  // namespace rnd
