// rays.cuh — one LIDAR ray against one target (ref core.py:1281-1372, 1414-1490, 1544-1626).  Shared by the ray
// kernels of vmas_b200.cu (cast_rays_kernel, cast_rays_batched_kernel), the LIDAR stage of the whole-step kernel's
// epilogue (spec_lidar in spec_kernel.cuh) and the CPU harness of tests/hostsim: one set of functions, so every route
// casts a ray with the same arithmetic in the same order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "geometry.cuh"
#include "vmas_b200.h"

namespace vmas {

// torch.min / torch.max propagate NaN; fminf / fmaxf do not.
DEVI float tmin(float x, float y) { return (x != x || y != y) ? NAN : fminf(x, y); }
DEVI float tmax(float x, float y) { return (x != x || y != y) ? NAN : fmaxf(x, y); }

// ref core.py:1414-1490
DEVI float ray_vs_sphere(V2 o, float dc, float ds, V2 c, float radius, float max_range) {
  const float half = max_range / 2.f;
  V2 line_pos = mk(o.x + dc * half, o.y + ds * half);
  V2 u = c - o;
  if (!((u.x * dc + u.y * ds) > 0.f)) return max_range;  // behind the sensor
  V2 closest = closest_point_carrier(line_pos, dc, ds, c);
  float dn = norm2(c - closest);
  if (!(dn < radius)) return max_range;  // the carrier passes the sphere by
  float aa = radius * radius - dn * dn;
  float m = sqrtf(aa > 0.f ? aa : 1e-8f);
  return norm2(closest - o) - m;
}

// The ray from `o` along (dc, ds) against one target.  `t` is the caller's view of the target: shape() (VMAS_SHAPE_*),
// pos(), rot(), d0() (radius or length), d1() (width), each called where the shape needs it — loads from the tables
// and the slab in the ray kernels, registers and compile-time constants in the whole-step kernel.
template <class T>
DEVI float ray_vs_shape(const T& t, V2 o, float dc, float ds, float max_range) {
  const int shape = t.shape();
  const V2 c = t.pos();
  if (shape == VMAS_SHAPE_SPHERE) return ray_vs_sphere(o, dc, ds, c, t.d0(), max_range);
  const float trot = t.rot();
  if (shape == VMAS_SHAPE_BOX) {
    const float L = t.d0(), Wd = t.d1();
    float sn, cs;
    sincosf(-trot, &sn, &cs);
    V2 ol = rot2(o - c, cs, sn);
    V2 dl = rot2(mk(dc, ds), cs, sn);
    float tx1 = (-L / 2.f - ol.x) / dl.x, tx2 = (L / 2.f - ol.x) / dl.x;
    float t0 = tmin(tx1, tx2), t1 = tmax(tx1, tx2);
    float ty1 = (-Wd / 2.f - ol.y) / dl.y, ty2 = (Wd / 2.f - ol.y) / dl.y;
    float ty0 = tmin(ty1, ty2), tyM = tmax(ty1, ty2);
    t0 = tmax(t0, ty0);
    t1 = tmin(t1, tyM);
    V2 hl = mk(t0 * dl.x + ol.x, t0 * dl.y + ol.y);
    float sn2, cs2;
    sincosf(trot, &sn2, &cs2);
    V2 hw = rot2(hl, cs2, sn2) + c;
    bool hit = (t1 >= t0) && (t0 > 0.f);
    return hit ? norm2(o - hw) : max_range;
  }
  // line
  {
    const float L = t.d0();
    float sn, cs;
    sincosf(trot, &sn, &cs);
    V2 r = mk(cs * L, sn * L);
    V2 s = mk(dc, ds);
    float rxs = cross2(r, s);
    V2 qp = o - c;
    float tt = cross2(qp, mk(s.x / rxs, s.y / rxs));
    float uu = cross2(qp, mk(r.x / rxs, r.y / rxs));
    float d = norm2(uu * s.x, uu * s.y);
    bool miss = (rxs == 0.f) || (tt > 0.5f) || (tt < -0.5f) || (uu < 0.f);
    return miss ? max_range : d;
  }
}

// Exact early-out shared by every ray route: a target centred at `c` whose circumscribed circle (radius `circ_r`) lies
// beyond the sensor's range cannot shorten a ray (any hit distance is >= |c - o| - circ_r > max_range, and the result
// is min(max_range, ...)), so its shape test — and, when no target is in reach, the ray's sin/cos — is skipped.  The
// margin dwarfs fp32 rounding of the skipped arithmetic.
DEVI bool ray_in_reach(V2 o, V2 c, float circ_r, float max_range) {
  const float reach = (max_range + circ_r) * 1.001f + 1e-3f;
  const float dx = c.x - o.x, dy = c.y - o.y;
  return !(dx * dx + dy * dy > reach * reach);  // NaN positions stay "in reach"
}

// ---- the ray kernels' view: targets in the plan tables and the state slab ------------------------------------------
struct RayArgs {
  VmasWorldConfig cfg;
  VmasPlanTables tb;
  VmasState st;
  const int32_t* targets;
  const float* angles;
  float* out;
  int32_t src, n_targets, n_rays, add_rot_of;
  float max_range;
};

// target t of the env at env_base in the plan tables and the state slab: its shape, table row and position taken up
// front, its heading and sizes loaded where a shape reads them (the ray kernels' order of loads).  Templates on the
// arguments' type (RayArgs) only so that a host build of the headers needs no __ldg unless it calls them.
template <class A>
struct RayTableTarget {
  const A& a;
  int t;
  size_t env_base;
  int shape_;
  decltype(A::tb.ent_f32) ef;  // the entity's row of the table
  V2 c;
  DEVI int shape() const { return shape_; }
  DEVI V2 pos() const { return c; }
  DEVI float rot() const { return a.st.rot[env_base + t]; }
  DEVI float d0() const { return __ldg(ef + VMAS_EF_D0); }
  DEVI float d1() const { return __ldg(ef + VMAS_EF_D1); }
};

template <class A>
DEVI float ray_vs_entity(const A& a, V2 o, float ang, float dc, float ds, int t, size_t env_base) {
  const int shape = __ldg(a.tb.ent_i32 + t * 4);
  const float* ef = a.tb.ent_f32 + (size_t)t * VMAS_EF_COLS;
  const float2 tp = reinterpret_cast<const float2*>(a.st.pos)[env_base + t];
  return ray_vs_shape(RayTableTarget<A>{a, t, env_base, shape, ef, mk(tp.x, tp.y)}, o, dc, ds, a.max_range);
}

template <class A>
DEVI bool ray_target_in_reach(const A& a, V2 o, int t, size_t env_base) {
  const float2 tp = reinterpret_cast<const float2*>(a.st.pos)[env_base + t];
  return ray_in_reach(o, mk(tp.x, tp.y), __ldg(a.tb.ent_f32 + (size_t)t * VMAS_EF_COLS + VMAS_EF_CIRC_R), a.max_range);
}

}  // namespace vmas
