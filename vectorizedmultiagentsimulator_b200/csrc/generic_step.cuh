// generic_step.cuh — the per-env arithmetic of the generic (unspecialised) substep kernels: the kernel
// arguments, the work-item evaluation, and the per-entity phases of a substep (forces before the work
// items, integration after them).  Included by vmas_b200.cu (step_kernel, step_tpe_kernel,
// step_block_kernel); tests/hostsim compiles it with g++ and runs the phases on the CPU.
//
// The phases read and write an env's state through `col` and a compile-time PITCH (field k of the T_*
// enum, entity e at col[(k * E + e) * PITCH]): the thread-per-env kernel keeps the state as
// [field][entity][thread], the block-per-env kernel as [field][entity].  Every function performs its
// statements in the same order whatever the layout, so the two kernels produce the same bits.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "geometry.cuh"
#include "vmas_b200.h"

namespace vmas {

constexpr float HALF_PI_F = 1.57079632679489661923f;  // fp32(torch.pi / 2)

struct StepArgs {
  VmasWorldConfig cfg;
  VmasPlanTables tb;
  VmasState st;
  uint32_t* mask;      // [mask_words + 1]; last word counts blocks that have consumed the mask
  int use_mask;
  int mask_words;
  int first_substep;
  int n_substeps;
  const float* ent_params = nullptr;  // [B, E, VMAS_EP_COLS] per-env mass / friction of flagged entities, or null
};

// an entity's per-env parameter (VMAS_F_*_ENV flag `bit`, column `col` of ent_params) or its scalar column
DEVI float ent_param(const StepArgs& a, int flg, int bit, long env, int e, int col, const float* ef, int ef_col) {
  return ((flg & bit) && a.ent_params) ? a.ent_params[((size_t)env * a.cfg.n_entities + e) * VMAS_EP_COLS + col]
                                       : __ldg(ef + ef_col);
}
// moment of inertia: per env from the env's mass (VMAS_F_MASS_ENV), else the scalar column
DEVI float ent_inertia(const StepArgs& a, int flg, float mass, const float* ef) {
  return ((flg & VMAS_F_MASS_ENV) && a.ent_params)
             ? (__ldg(ef + VMAS_EF_INERTIA_K0) * mass) * __ldg(ef + VMAS_EF_INERTIA_K1)
             : __ldg(ef + VMAS_EF_INERTIA);
}

// ---------------------------------------------------------------------------------------------
// per-entity geometry cached in shared memory for the work-item phase
// ---------------------------------------------------------------------------------------------
// PITCH = distance (in floats) between consecutive entities of one env: 1 when a group of lanes or a
// block owns an env (entity-major slice per env), blockDim when one thread owns an env (the thread
// index is the fastest-varying dimension, so a warp reads 32 consecutive words: no bank conflicts).
template <int PITCH>
struct EnvShared {
  float *px, *py, *rot, *c, *s, *c2, *s2;  // per-entity geometry of this env
  float *rfx, *rfy, *rta, *rtb;            // per-item results (lane-per-entity kernel only)
  int pitch;                               // runtime pitch when PITCH == 0
  DEVI int at(int e) const { return PITCH ? e * PITCH : e * pitch; }
};

template <int PITCH>
DEVI V2 ent_pos(const EnvShared<PITCH>& sh, int e) { return mk(sh.px[sh.at(e)], sh.py[sh.at(e)]); }

template <int PITCH>
DEVI Seg ent_seg(const EnvShared<PITCH>& sh, int e, float length) {
  return mkseg(ent_pos(sh, e), sh.c[sh.at(e)], sh.s[sh.at(e)], length / 2.f);
}

template <int PITCH>
DEVI BoxG ent_box(const EnvShared<PITCH>& sh, int e, float length, float width) {
  BoxG b;
  b.p = ent_pos(sh, e);
  b.c = sh.c[sh.at(e)];
  b.s = sh.s[sh.at(e)];
  b.c2 = sh.c2[sh.at(e)];
  b.s2 = sh.s2[sh.at(e)];
  b.half_l = length / 2.f;
  b.half_w = width / 2.f;
  return b;
}

// Conservative rejection used before the narrow phase.  A contact force is non-zero only while the
// two shapes are within their contact threshold of each other; when even the bounding regions are
// farther apart than that threshold plus FAR_MARGIN (>> any fp32 rounding of these coordinates)
// the reference's result is an exact 0, which is what skipping produces.
constexpr float FAR_MARGIN = 1e-3f;
DEVI bool far_apart(V2 a, V2 b, float reach) {
  V2 d = a - b;
  float lim = reach + FAR_MARGIN;
  return d.x * d.x + d.y * d.y > lim * lim;
}

// One work item -> (force on a, torque on a, torque on b); the force on b is the negative.
template <int PITCH>
DEVI void eval_item(const StepArgs& a, const EnvShared<PITCH>& sh, int item, long env, float* out_fx,
                    float* out_fy, float* out_ta, float* out_tb) {
  const int4 ii = __ldg(reinterpret_cast<const int4*>(a.tb.item_i32) + item);
  const int kind = ii.x, ea = ii.y, eb = ii.z, flags = ii.w & 0xff;
  const float* f32 = a.tb.item_f32 + (size_t)item * VMAS_IF_COLS;
  const float dmin_base = __ldg(f32 + VMAS_IF_DMIN_BASE);
  const float* pa_f = a.tb.ent_f32 + (size_t)ea * VMAS_EF_COLS;
  const float* pb_f = a.tb.ent_f32 + (size_t)eb * VMAS_EF_COLS;
  const float cf = a.cfg.collision_force, km = a.cfg.contact_margin;
  V2 f = mk(0.f, 0.f);
  float ta = 0.f, tb = 0.f;

  switch (kind) {
    case VMAS_K_JOINT: {  // ref core.py:2201-2292, joints.py:209-216
      V2 pa = ent_pos(sh, ea), pb = ent_pos(sh, eb);
      V2 da = mk(__ldg(f32 + VMAS_IF_AX), __ldg(f32 + VMAS_IF_AY));
      V2 db = mk(__ldg(f32 + VMAS_IF_BX), __ldg(f32 + VMAS_IF_BY));
      V2 qa = pa + rot2(da, sh.c[sh.at(ea)], sh.s[sh.at(ea)]);
      V2 qb = pb + rot2(db, sh.c[sh.at(eb)], sh.s[sh.at(eb)]);
      float dist = __ldg(f32 + VMAS_IF_DIST);
      V2 f_attr = constraint_force(qa, qb, dist, a.cfg.joint_force, km, true);
      V2 f_rep = constraint_force(qa, qb, dist, a.cfg.joint_force, km, false);
      f = f_attr + f_rep;
      V2 fb = neg(f_attr) + neg(f_rep);
      ta = cross2(qa - pa, f);
      tb = cross2(qb - pb, fb);
      if (!(flags & VMAS_IFLAG_JOINT_ROTATE)) {  // ref core.py:2841-2858
        float jr = (flags & VMAS_IFLAG_JOINT_ROT_PER_ENV)
                       ? a.tb.joint_rot[(size_t)env * a.cfg.n_joints + item]
                       : __ldg(f32 + VMAS_IF_FIXED_ROT);
        float ra = sh.rot[sh.at(ea)], rb = sh.rot[sh.at(eb)];
        float delta = ra - (rb + jr);
        float mag = sqrtf(delta * delta);
        float t = (a.cfg.torque_constraint_force * sgnf(delta)) * (expf(mag) - 1.f);
        if (mag < 1e-9f) t = 0.f;
        ta = ta + (-t);
        tb = tb + t;
      }
      break;
    }
    case VMAS_K_SS: {  // ref core.py:2294-2339
      f = constraint_force(ent_pos(sh, ea), ent_pos(sh, eb), dmin_base, cf, km, false);
      break;
    }
    case VMAS_K_LS: {  // a = line, b = sphere; ref core.py:2341-2392
      Seg l = ent_seg(sh, ea, __ldg(pa_f + VMAS_EF_D0));
      V2 ps = ent_pos(sh, eb);
      if (far_apart(l.p, ps, l.half + dmin_base)) break;
      V2 cp = closest_point_seg(l, ps);
      V2 f_sphere = constraint_force(ps, cp, dmin_base, cf, km, false);
      f = neg(f_sphere);  // force on the line
      ta = cross2(cp - l.p, f);
      break;
    }
    case VMAS_K_LL: {  // ref core.py:2394-2457
      Seg l1 = ent_seg(sh, ea, __ldg(pa_f + VMAS_EF_D0));
      Seg l2 = ent_seg(sh, eb, __ldg(pb_f + VMAS_EF_D0));
      if (far_apart(l1.p, l2.p, l1.half + l2.half + dmin_base)) break;
      Pair c = closest_seg_seg(l1, l2);
      f = constraint_force(c.a, c.b, dmin_base, cf, km, false);
      ta = cross2(c.a - l1.p, f);
      tb = cross2(c.b - l2.p, neg(f));
      break;
    }
    case VMAS_K_BS: {  // a = box, b = sphere; ref core.py:2459-2552
      BoxG bx = ent_box(sh, ea, __ldg(pa_f + VMAS_EF_D0), __ldg(pa_f + VMAS_EF_D1));
      const bool hollow = __ldg(a.tb.ent_i32 + ea * 4 + 1) & VMAS_F_HOLLOW;
      V2 ps = ent_pos(sh, eb);
      {  // sphere centre outside the box inflated by r + LINE_MIN_DIST (+ margin): force is exactly 0
        V2 d = ps - bx.p;
        float lx = d.x * bx.c + d.y * bx.s, ly = d.y * bx.c - d.x * bx.s;
        if (fabsf(lx) > bx.half_l + dmin_base + FAR_MARGIN || fabsf(ly) > bx.half_w + dmin_base + FAR_MARGIN) break;
      }
      V2 cp = closest_point_box(bx, ps);
      V2 inner = cp;
      float d = 0.f;
      if (!hollow) inner = inner_point_box(ps, cp, bx.p, &d);
      V2 f_sphere = constraint_force(ps, inner, dmin_base + d, cf, km, false);
      f = neg(f_sphere);  // force on the box
      ta = cross2(cp - bx.p, f);
      break;
    }
    case VMAS_K_BL: {  // a = box, b = line; ref core.py:2554-2653
      BoxG bx = ent_box(sh, ea, __ldg(pa_f + VMAS_EF_D0), __ldg(pa_f + VMAS_EF_D1));
      const bool hollow = __ldg(a.tb.ent_i32 + ea * 4 + 1) & VMAS_F_HOLLOW;
      Seg l = ent_seg(sh, eb, __ldg(pb_f + VMAS_EF_D0));
      {  // segment entirely outside the box inflated by LINE_MIN_DIST (+ margin): force is exactly 0
        V2 d = l.p - bx.p;
        float lx = d.x * bx.c + d.y * bx.s, ly = d.y * bx.c - d.x * bx.s;
        float ex = l.half * fabsf(l.c * bx.c + l.s * bx.s), ey = l.half * fabsf(l.s * bx.c - l.c * bx.s);
        if (fabsf(lx) - ex > bx.half_l + dmin_base + FAR_MARGIN || fabsf(ly) - ey > bx.half_w + dmin_base + FAR_MARGIN)
          break;
      }
      Pair c = closest_box_seg(bx, l);
      V2 inner = c.a;
      float d = 0.f;
      if (!hollow) inner = inner_point_box(c.b, c.a, bx.p, &d);
      f = constraint_force(inner, c.b, dmin_base + d, cf, km, false);
      ta = cross2(c.a - bx.p, f);
      tb = cross2(c.b - l.p, neg(f));
      break;
    }
    case VMAS_K_BB: {  // ref core.py:2655-2786
      BoxG b1 = ent_box(sh, ea, __ldg(pa_f + VMAS_EF_D0), __ldg(pa_f + VMAS_EF_D1));
      BoxG b2 = ent_box(sh, eb, __ldg(pb_f + VMAS_EF_D0), __ldg(pb_f + VMAS_EF_D1));
      const bool hollow1 = __ldg(a.tb.ent_i32 + ea * 4 + 1) & VMAS_F_HOLLOW;
      const bool hollow2 = __ldg(a.tb.ent_i32 + eb * 4 + 1) & VMAS_F_HOLLOW;
      if (far_apart(b1.p, b2.p, __ldg(pa_f + VMAS_EF_CIRC_R) + __ldg(pb_f + VMAS_EF_CIRC_R) + dmin_base)) break;
      Pair c = closest_box_box(b1, b2);
      V2 in1 = c.a, in2 = c.b;
      float d1 = 0.f, d2 = 0.f;
      if (!hollow1) in1 = inner_point_box(c.b, c.a, b1.p, &d1);
      if (!hollow2) in2 = inner_point_box(c.a, c.b, b2.p, &d2);
      f = constraint_force(in1, in2, (d1 + d2) + dmin_base, cf, km, false);
      ta = cross2(c.a - b1.p, f);
      tb = cross2(c.b - b2.p, neg(f));
      break;
    }
    default:
      break;
  }
  *out_fx = f.x;
  *out_fy = f.y;
  *out_ta = ta;
  *out_tb = tb;
}

// ---------------------------------------------------------------------------------------------
// the per-entity phases of a substep on an env's state held in shared memory
// ---------------------------------------------------------------------------------------------
enum { T_PX = 0, T_PY, T_ROT, T_C, T_S, T_C2, T_S2, T_VX, T_VY, T_W, T_FX, T_FY, T_TQ, T_NF };

// Field k of entity e of the env: col[(k * E + e) * PITCH].  PITCH = the block size for the thread-per-env
// kernel ([field][entity][thread], `col` = the thread's column), 1 for the block-per-env kernel
// ([field][entity]).
#define GS_F(k, e) col[((k)*E + (e)) * PITCH]

// Phase A for entity e: trig cache and the per-entity forces (ref core.py:1995-2004): the agent's
// clamped action force / torque (written back to the agent's rows), friction, gravity.
template <int PITCH>
DEVI void entity_forces(const StepArgs& a, float* col, int E, int e, long env, size_t ebase, size_t abase, float sub_dt) {
  const int flg = __ldg(a.tb.ent_i32 + e * 4 + 1);
  const float* ef = a.tb.ent_f32 + (size_t)e * VMAS_EF_COLS;
  if (flg & VMAS_F_TRIG) {
    const float r = GS_F(T_ROT, e);
    float sn, cs;
    sincosf(r, &sn, &cs);
    GS_F(T_C, e) = cs;
    GS_F(T_S, e) = sn;
    if (__ldg(a.tb.ent_i32 + e * 4) == VMAS_SHAPE_BOX) {
      sincosf(r + HALF_PI_F, &sn, &cs);
      GS_F(T_C2, e) = cs;
      GS_F(T_S2, e) = sn;
    }
  }
  float Fx = 0.f, Fy = 0.f, T = 0.f;
  const float mass = ent_param(a, flg, VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS);
  if (flg & VMAS_F_AGENT) {  // ref core.py:2018-2041
    const int ai = __ldg(a.tb.ent_i32 + e * 4 + 2);
    if (flg & VMAS_F_MOVABLE) {
      float2 af = reinterpret_cast<const float2*>(a.st.force)[abase + ai];
      if (flg & (VMAS_F_MAX_F | VMAS_F_F_RANGE)) {
        if (flg & VMAS_F_MAX_F) {
          const float mx = __ldg(ef + VMAS_EF_MAX_F);
          const float n = norm2(af.x, af.y);
          if (n > mx) {
            af.x = (af.x / n) * mx;
            af.y = (af.y / n) * mx;
          }
        }
        if (flg & VMAS_F_F_RANGE) {
          const float r = __ldg(ef + VMAS_EF_F_RANGE);
          af.x = clampf(af.x, -r, r);
          af.y = clampf(af.y, -r, r);
        }
        reinterpret_cast<float2*>(a.st.force)[abase + ai] = af;
      }
      Fx = Fx + af.x;
      Fy = Fy + af.y;
    }
    if (flg & VMAS_F_ROTATABLE) {
      float tq = a.st.torque[abase + ai];
      if (flg & (VMAS_F_MAX_T | VMAS_F_T_RANGE)) {
        if (flg & VMAS_F_MAX_T) {
          const float mx = __ldg(ef + VMAS_EF_MAX_T);
          const float n = fabsf(tq);  // vector_norm of one element
          if (n > mx) tq = (tq / n) * mx;
        }
        if (flg & VMAS_F_T_RANGE) {
          const float r = __ldg(ef + VMAS_EF_T_RANGE);
          tq = clampf(tq, -r, r);
        }
        a.st.torque[abase + ai] = tq;
      }
      T = T + tq;
    }
  }
  if (flg & VMAS_F_LIN_FRIC) {  // ref core.py:2054-2088
    const float vx = GS_F(T_VX, e), vy = GS_F(T_VY, e);
    const float speed = norm2(vx, vy);
    if (speed != 0.f) {
      const float cap = ent_param(a, flg, VMAS_F_LIN_FRIC_ENV, env, e, VMAS_EP_LIN_FRIC, ef, VMAS_EF_LIN_FRIC) * mass;
      Fx = Fx + (-(vx / speed)) * fminf(cap, (fabsf(vx) / sub_dt) * mass);
      Fy = Fy + (-(vy / speed)) * fminf(cap, (fabsf(vy) / sub_dt) * mass);
    }
  }
  if (flg & VMAS_F_ANG_FRIC) {  // ref core.py:2089-2102
    const float w = GS_F(T_W, e);
    const float speed = fabsf(w);  // vector_norm of one element
    if (speed != 0.f) {
      const float inertia = ent_inertia(a, flg, mass, ef);
      const float cap = ent_param(a, flg, VMAS_F_ANG_FRIC_ENV, env, e, VMAS_EP_ANG_FRIC, ef, VMAS_EF_ANG_FRIC) * inertia;
      T = T + (-(w / speed)) * fminf(cap, (fabsf(w) / sub_dt) * inertia);
    }
  }
  if (flg & VMAS_F_MOVABLE) {  // ref core.py:2043-2052
    if (a.cfg.has_world_gravity) {
      Fx = Fx + mass * a.cfg.gravity_x;
      Fy = Fy + mass * a.cfg.gravity_y;
    }
    if (flg & VMAS_F_GRAVITY) {
      Fx = Fx + mass * __ldg(ef + VMAS_EF_GRAV_X);
      Fy = Fy + mass * __ldg(ef + VMAS_EF_GRAV_Y);
    }
    if (flg & VMAS_F_GRAVITY_ENV) {
      const float2 g = reinterpret_cast<const float2*>(a.tb.ent_gravity)[ebase + e];
      Fx = Fx + mass * g.x;
      Fy = Fy + mass * g.y;
    }
  }
  GS_F(T_FX, e) = Fx;
  GS_F(T_FY, e) = Fy;
  GS_F(T_TQ, e) = T;
}

// the batch-wide broad phase switched this item off (ref core.py:2797-2801)
DEVI bool item_masked_off(const StepArgs& a, const uint32_t* s_mask, int item_w) {
  if (!a.use_mask) return false;
  const int mbit = (item_w >> 8) - 1;
  return mbit >= 0 && !((s_mask[mbit >> 5] >> (mbit & 31)) & 1u);
}

// Phase B in item order (the thread-per-env kernel): item `item` evaluated once, its force and torque
// added to both entities' accumulators.
template <int PITCH>
DEVI void item_accumulate(const StepArgs& a, const EnvShared<PITCH>& sh, float* col, int E, int item, long env,
                          const uint32_t* s_mask) {
  const int4 ii = __ldg(reinterpret_cast<const int4*>(a.tb.item_i32) + item);
  if (a.use_mask) {  // (item_masked_off spelled out: calling it changes step_tpe_kernel's instruction schedule)
    const int mbit = (ii.w >> 8) - 1;
    if (mbit >= 0 && !((s_mask[mbit >> 5] >> (mbit & 31)) & 1u)) return;
  }
  float fx, fy, ta, tb;
  eval_item(a, sh, item, env, &fx, &fy, &ta, &tb);
  const int fa = __ldg(a.tb.ent_i32 + ii.y * 4 + 1), fb = __ldg(a.tb.ent_i32 + ii.z * 4 + 1);
  if (fa & VMAS_F_MOVABLE) {
    GS_F(T_FX, ii.y) = GS_F(T_FX, ii.y) + fx;
    GS_F(T_FY, ii.y) = GS_F(T_FY, ii.y) + fy;
  }
  if (fa & VMAS_F_ROTATABLE) GS_F(T_TQ, ii.y) = GS_F(T_TQ, ii.y) + ta;
  if (fb & VMAS_F_MOVABLE) {
    GS_F(T_FX, ii.z) = GS_F(T_FX, ii.z) + (-fx);
    GS_F(T_FY, ii.z) = GS_F(T_FY, ii.z) + (-fy);
  }
  if (fb & VMAS_F_ROTATABLE) GS_F(T_TQ, ii.z) = GS_F(T_TQ, ii.z) + tb;
}

// Phase B in entity order (the block-per-env kernel): entity e walks its incidence list
// inc[inc_off[e] .. inc_off[e + 1]) — its items in ascending order, each with the side e is on — and
// adds its own side of every active item.  That is the item-order walk's sequence of additions into
// e's accumulators, operand for operand, so both produce the same bits.
template <int PITCH>
DEVI void entity_accumulate(const StepArgs& a, const EnvShared<PITCH>& sh, float* col, int E, int e, long env,
                            const uint32_t* s_mask) {
  const int flg = __ldg(a.tb.ent_i32 + e * 4 + 1);
  const bool movable = flg & VMAS_F_MOVABLE, rotatable = flg & VMAS_F_ROTATABLE;
  if (!movable && !rotatable) return;
  float Fx = GS_F(T_FX, e), Fy = GS_F(T_FY, e), T = GS_F(T_TQ, e);
  const int lo = __ldg(a.tb.inc_off + e), hi = __ldg(a.tb.inc_off + e + 1);
  for (int i = lo; i < hi; ++i) {
    const int v = __ldg(a.tb.inc + i);
    const int item = v >> 1;
    if (item_masked_off(a, s_mask, __ldg(a.tb.item_i32 + item * 4 + 3))) continue;
    float fx, fy, ta, tb;
    eval_item(a, sh, item, env, &fx, &fy, &ta, &tb);
    if (v & 1) {
      if (movable) {
        Fx = Fx + (-fx);
        Fy = Fy + (-fy);
      }
      if (rotatable) T = T + tb;
    } else {
      if (movable) {
        Fx = Fx + fx;
        Fy = Fy + fy;
      }
      if (rotatable) T = T + ta;
    }
  }
  GS_F(T_FX, e) = Fx;
  GS_F(T_FY, e) = Fy;
  GS_F(T_TQ, e) = T;
}

// Phase C for entity e: semi-implicit Euler (ref core.py:2862-2908) with drag on the first substep,
// max_speed / v_range and the world's semidims.
template <int PITCH>
DEVI void entity_integrate(const StepArgs& a, float* col, int E, int e, long env, int sub, float sub_dt) {
  const int flg = __ldg(a.tb.ent_i32 + e * 4 + 1);
  if (!(flg & (VMAS_F_MOVABLE | VMAS_F_ROTATABLE))) return;
  const float* ef = a.tb.ent_f32 + (size_t)e * VMAS_EF_COLS;
  const float drag_mult = __ldg(ef + VMAS_EF_DRAG_MULT);
  if (flg & VMAS_F_MOVABLE) {
    const float mass = ent_param(a, flg, VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS);
    float vx = GS_F(T_VX, e), vy = GS_F(T_VY, e);
    if (sub == 0) {
      vx = vx * drag_mult;
      vy = vy * drag_mult;
    }
    vx = vx + div_pos(GS_F(T_FX, e), mass) * sub_dt;
    vy = vy + div_pos(GS_F(T_FY, e), mass) * sub_dt;
    if (flg & VMAS_F_MAX_SPEED) {
      const float mx = __ldg(ef + VMAS_EF_MAX_SPEED);
      const float n = norm2(vx, vy);
      if (n > mx) {
        vx = (vx / n) * mx;
        vy = (vy / n) * mx;
      }
    }
    if (flg & VMAS_F_V_RANGE) {
      const float r = __ldg(ef + VMAS_EF_V_RANGE);
      vx = clampf(vx, -r, r);
      vy = clampf(vy, -r, r);
    }
    float px = GS_F(T_PX, e) + vx * sub_dt;
    float py = GS_F(T_PY, e) + vy * sub_dt;
    if (a.cfg.has_x_semidim) px = clampf(px, -a.cfg.x_semidim, a.cfg.x_semidim);
    if (a.cfg.has_y_semidim) py = clampf(py, -a.cfg.y_semidim, a.cfg.y_semidim);
    GS_F(T_VX, e) = vx;
    GS_F(T_VY, e) = vy;
    GS_F(T_PX, e) = px;
    GS_F(T_PY, e) = py;
  }
  if (flg & VMAS_F_ROTATABLE) {
    const float inertia =
        ent_inertia(a, flg, ent_param(a, flg, VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS), ef);
    float w = GS_F(T_W, e);
    if (sub == 0) w = w * drag_mult;
    w = w + div_pos(GS_F(T_TQ, e), inertia) * sub_dt;
    GS_F(T_W, e) = w;
    GS_F(T_ROT, e) = GS_F(T_ROT, e) + w * sub_dt;
  }
}

// Slab rows of entity e -> the env's shared state (velocities of static bodies read as 0).
template <int PITCH>
DEVI void entity_load(const StepArgs& a, float* col, int E, int e, size_t ebase) {
  const int flg = __ldg(a.tb.ent_i32 + e * 4 + 1);
  const float2 p = reinterpret_cast<const float2*>(a.st.pos)[ebase + e];
  GS_F(T_PX, e) = p.x;
  GS_F(T_PY, e) = p.y;
  GS_F(T_ROT, e) = a.st.rot[ebase + e];
  float2 v = make_float2(0.f, 0.f);
  if (flg & VMAS_F_MOVABLE) v = reinterpret_cast<const float2*>(a.st.vel)[ebase + e];
  GS_F(T_VX, e) = v.x;
  GS_F(T_VY, e) = v.y;
  GS_F(T_W, e) = (flg & VMAS_F_ROTATABLE) ? a.st.ang_vel[ebase + e] : 0.f;
}

// The env's shared state of entity e -> its slab rows: only what can have changed.
template <int PITCH>
DEVI void entity_store(const StepArgs& a, float* col, int E, int e, size_t ebase) {
  const int flg = __ldg(a.tb.ent_i32 + e * 4 + 1);
  if (flg & VMAS_F_MOVABLE) {
    reinterpret_cast<float2*>(a.st.pos)[ebase + e] = make_float2(GS_F(T_PX, e), GS_F(T_PY, e));
    reinterpret_cast<float2*>(a.st.vel)[ebase + e] = make_float2(GS_F(T_VX, e), GS_F(T_VY, e));
  }
  if (flg & VMAS_F_ROTATABLE) {
    a.st.rot[ebase + e] = GS_F(T_ROT, e);
    a.st.ang_vel[ebase + e] = GS_F(T_W, e);
  }
}

#undef GS_F

}  // namespace vmas
