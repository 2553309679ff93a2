// spec_kernel.cuh — world-specialised substep kernel.
//
// The generic kernels in vmas_b200.cu interpret the plan tables at run time (table loads,
// dynamically indexed shared memory, a switch per work item) and end up latency-bound.  Here the
// world's static structure is a compile-time constant: a generated header (csrc/generated/) holds
// one `struct World_<hash>` per pre-registered world with constexpr entity / item tables, and this
// template unrolls every loop over entities and work items.  After unrolling all indices are
// constants, so an env's whole state (positions, velocities, rotations, force accumulators, cached
// sin/cos) lives in REGISTERS of the one thread that owns the env, shape parameters fold into
// immediates, and the kind dispatch disappears.  The arithmetic is the same device functions
// (geometry.cuh) in the same order as the generic kernels: results are bit-identical (tested).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>
#include <utility>

#include "geometry.cuh"
#include "ingest.cuh"
#include "query.cuh"
#include "rays.cuh"
#include "vmas_b200.h"

namespace vmas {

struct EntC {
  int shape, flags, agent;
  float d0, d1, mass, inertia, drag_mult, lin_fric, ang_fric, grav_x, grav_y, max_speed, v_range, max_f, f_range,
      max_t, t_range, circ_r, r_plus_lmd;
  float inertia_k0, inertia_k1;  // (worlds with per-env masses only: see SpecEnvParams)
};
struct ItemC {
  int kind, a, b, flags, mask_bit;
  float dmin_base, ax, ay, bx, by, dist, fixed_rot, broad_thr;
};
struct CfgC {
  int substeps, has_x_semidim, has_y_semidim, has_world_gravity;
  float sub_dt, x_semidim, y_semidim, collision_force, joint_force, torque_constraint_force, contact_margin,
      gravity_x, gravity_y;
};

// The whole-step kernel's epilogue (see spec_epilogue): the scenario's step program and observation rows,
// compile-time data like the world itself
struct ProgC {
  int op, dst, a, b, arg;
  float imm;
};
struct ObsColC {
  int op, src, src2;  // as the observation gather's column codes: (field << 24) | element offset in the env's row
  float par;
};
// ... and its LIDAR stage (see spec_lidar): one sensor of the plan, its angles in P::lidar_angle
constexpr int SPEC_LIDAR_MAX_TARGETS = 16;  // (codegen.MAX_LIDAR_TARGETS: a plan with more stays on the captured graph)
static_assert(SPEC_LIDAR_MAX_TARGETS <= 32, "spec_lidar keeps a sensor's targets in reach as bits of one word");
struct LidarC {
  int src, row, col;  // the sensor's entity; its observation row and first column
  float max_range;
  int n_targets;
  int target[SPEC_LIDAR_MAX_TARGETS];  // the entities its rays can hit, in backend.ray_targets order
};
struct EpiArgs {
  void* obs_out;  // [rows, B, width] of P::OBS_DTYPE (fp32, fp16 or bf16), or null
  void* buffers[VMAS_PROG_MAX_BUFFERS];
};
// ... and its prologue (see spec_ingest_lane, spec_act_lane): the policy agents' actions, continuous, discrete or
// multi-discrete, through their action model (holonomic, with rotation, forward, rotation, differential drive)
struct ActC {
  int agent;  // row of the agent in the force / torque slab
  float range0, range1, mult0, mult1;
  int kind = VMAS_ACT_CONTINUOUS;  // VMAS_ACT_*
  int n0 = 0, n1 = 0;              // (discrete kinds) choices per component
  int dyn = VMAS_DYN_HOLONOMIC;    // VMAS_DYN_*
  int size = 2;                    // action components: the model's own, 1-4
  float range2 = 0.f, range3 = 0.f, mult2 = 0.f, mult3 = 0.f;
  int n2 = 0, n3 = 0;
  float params[8] = {};  // the model's parameters (VmasAgentActions::dyn_params)
};
// a holonomic agent with 2 components: its rounds run the lean decode of spec_ingest_lane
__host__ __device__ constexpr bool act_holonomic2(const ActC& c) { return c.dyn == VMAS_DYN_HOLONOMIC && c.size == 2; }
__host__ __device__ constexpr float act_range(const ActC& c, int j) {
  return j == 0 ? c.range0 : j == 1 ? c.range1 : j == 2 ? c.range2 : c.range3;
}
__host__ __device__ constexpr float act_mult(const ActC& c, int j) {
  return j == 0 ? c.mult0 : j == 1 ? c.mult1 : j == 2 ? c.mult2 : c.mult3;
}
__host__ __device__ constexpr int act_n(const ActC& c, int j) { return j == 0 ? c.n0 : j == 1 ? c.n1 : j == 2 ? c.n2 : c.n3; }
struct ActArgs {
  const float* actions[VMAS_MAX_INGEST_AGENTS];  // the caller's tensors: fp32 [B, size], or int64 [B, 1] / [B, size]
  float* u[VMAS_MAX_INGEST_AGENTS];              // [B, size] each: agent.action.u
  uint8_t* bad_flag;
  float* steps;  // [B] or null
  int clamp;
  // what each agent's tensors are (launch_env refuses a combination it was not built for): VMAS_ACT_*, VMAS_DYN_*,
  // the action size.  One byte each: the kernel never reads them, and every byte here is a byte of every launch.
  int8_t kind[VMAS_MAX_INGEST_AGENTS];
  int8_t dyn[VMAS_MAX_INGEST_AGENTS];
  int8_t size[VMAS_MAX_INGEST_AGENTS];
};
struct alignas(16) ActIdx2 {  // one multi-discrete env row, loaded as one 16-byte word
  long long i0, i1;
};

struct SpecArgs {
  VmasState st;
  const float* joint_rot;  // [B, n_joints] or null
  uint32_t* mask;          // [mask_words + 1]
  int batch_dim;
  int use_mask;
  int first_substep;
  int n_substeps;
  // env scheduling (optional, see vmas_b200_build_env_order): thread t steps env order[t]; every env
  // records which of its work items produced a force (bit I & 31) for the next re-ordering
  const int32_t* order;  // [B] permutation of the envs, or null: thread t steps env t
  uint32_t* sig;         // [B] out, or null
  // per-env physical parameters (worlds whose W::PER_ENV flags an entity only, see SpecEnvParams)
  const float* ent_params;   // [B, E, VMAS_EP_COLS]: mass, linear / angular friction coefficient, or null
  const float* ent_gravity;  // [B, E, 2], or null
};

template <class F, int... I>
DEVI void static_for_impl(F&& f, std::integer_sequence<int, I...>) {
  (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
DEVI void static_for(F&& f) {
  static_for_impl(static_cast<F&&>(f), std::make_integer_sequence<int, N>{});
}

constexpr float SPEC_HALF_PI_F = 1.57079632679489661923f;
constexpr float SPEC_FAR_MARGIN = 1e-3f;

DEVI bool spec_far_apart(V2 a, V2 b, float reach) {
  V2 d = a - b;
  float lim = reach + SPEC_FAR_MARGIN;
  return d.x * d.x + d.y * d.y > lim * lim;
}

// (x + y) + z with each sum rounded to float, as the kernel's run-time expressions round it
__host__ __device__ constexpr float spec_add3(float x, float y, float z) {
  const float s = x + y;
  return s + z;
}

// Register-resident state of one env.
template <int E>
struct EnvRegs {
  float px[E], py[E], rot[E], vx[E], vy[E], w[E];
  float c[E], s[E], c2[E], s2[E];
  float Fx[E], Fy[E], T[E];
};

template <class W, int EI, int E>
DEVI Seg spec_seg(const EnvRegs<E>& r) {
  return mkseg(mk(r.px[EI], r.py[EI]), r.c[EI], r.s[EI], W::ent[EI].d0 / 2.f);
}
template <class W, int EI, int E>
DEVI BoxG spec_box(const EnvRegs<E>& r) {
  BoxG b;
  b.p = mk(r.px[EI], r.py[EI]);
  b.c = r.c[EI];
  b.s = r.s[EI];
  b.c2 = r.c2[EI];
  b.s2 = r.s2[EI];
  b.half_l = W::ent[EI].d0 / 2.f;
  b.half_w = W::ent[EI].d1 / 2.f;
  return b;
}

// What one work item contributes: the force on `a` (`b` gets its negation) and the two torques
struct ItemOut {
  V2 f;
  float ta, tb;
};

// Two items run the same code (and may share a round of the lane-pair step, see SpecRounds): same kind, same
// mask gating, same joint rotation rule, same hollow flags.  Everything else differs only in constants.
template <class W>
__host__ __device__ constexpr bool spec_same_code(int i, int j) {
  const ItemC x = W::item[i], y = W::item[j];
  return x.kind == y.kind && (x.mask_bit >= 0) == (y.mask_bit >= 0) &&
         (x.flags & VMAS_IFLAG_JOINT_ROTATE) == (y.flags & VMAS_IFLAG_JOINT_ROTATE) &&
         (W::ent[x.a].flags & VMAS_F_HOLLOW) == (W::ent[y.a].flags & VMAS_F_HOLLOW) &&
         (W::ent[x.b].flags & VMAS_F_HOLLOW) == (W::ent[y.b].flags & VMAS_F_HOLLOW);
}

// One work item's contribution, fully resolved at compile time (ref core.py:2191-2199).  Item I0 on an even
// lane, I1 on an odd one (`odd`): the two must run the same code (spec_same_code), their entity indices and
// constants are picked by selects on the lane's parity, never by a run-time index into the register arrays.
// I0 == I1 (one lane per env, or a lone item): the selects fold away.
template <class W, int I0, int I1, int E>
DEVI ItemOut spec_item_eval(const EnvRegs<E>& r, const SpecArgs& a, long env, const bool odd) {
  static_assert(I0 == I1 || spec_same_code<W>(I0, I1), "the items of a round must run the same code");
  constexpr ItemC it = W::item[I0], jt = W::item[I1];
  constexpr int A0 = it.a, B0 = it.b, A1 = jt.a, B1 = jt.b;
  constexpr EntC ea = W::ent[A0], eb = W::ent[B0];  // (only their HOLLOW flags select code: same for both items)
  constexpr CfgC cfg = W::cfg;
  const bool o = I0 != I1 && odd;
  auto sel = [o](float x, float y) { return o ? y : x; };
  const float dmin = sel(it.dmin_base, jt.dmin_base);
  V2 f = mk(0.f, 0.f);
  float ta = 0.f, tb = 0.f;
  const V2 pa = mk(sel(r.px[A0], r.px[A1]), sel(r.py[A0], r.py[A1]));
  const V2 pb = mk(sel(r.px[B0], r.px[B1]), sel(r.py[B0], r.py[B1]));
  const float ca = sel(r.c[A0], r.c[A1]), sa = sel(r.s[A0], r.s[A1]);
  const float cb = sel(r.c[B0], r.c[B1]), sb = sel(r.s[B0], r.s[B1]);
  auto seg_a = [&]() { return mkseg(pa, ca, sa, sel(W::ent[A0].d0 / 2.f, W::ent[A1].d0 / 2.f)); };
  auto seg_b = [&]() { return mkseg(pb, cb, sb, sel(W::ent[B0].d0 / 2.f, W::ent[B1].d0 / 2.f)); };
  auto box_a = [&]() {
    BoxG b;
    b.p = pa;
    b.c = ca;
    b.s = sa;
    b.c2 = sel(r.c2[A0], r.c2[A1]);
    b.s2 = sel(r.s2[A0], r.s2[A1]);
    b.half_l = sel(W::ent[A0].d0 / 2.f, W::ent[A1].d0 / 2.f);
    b.half_w = sel(W::ent[A0].d1 / 2.f, W::ent[A1].d1 / 2.f);
    return b;
  };
  auto box_b = [&]() {
    BoxG b;
    b.p = pb;
    b.c = cb;
    b.s = sb;
    b.c2 = sel(r.c2[B0], r.c2[B1]);
    b.s2 = sel(r.s2[B0], r.s2[B1]);
    b.half_l = sel(W::ent[B0].d0 / 2.f, W::ent[B1].d0 / 2.f);
    b.half_w = sel(W::ent[B0].d1 / 2.f, W::ent[B1].d1 / 2.f);
    return b;
  };
  // the far-test bounds (half extent of `a` + dmin) + margin, folded per item
  constexpr float LIM_L0 = spec_add3(W::ent[A0].d0 / 2.f, it.dmin_base, SPEC_FAR_MARGIN);
  constexpr float LIM_L1 = spec_add3(W::ent[A1].d0 / 2.f, jt.dmin_base, SPEC_FAR_MARGIN);
  constexpr float LIM_W0 = spec_add3(W::ent[A0].d1 / 2.f, it.dmin_base, SPEC_FAR_MARGIN);
  constexpr float LIM_W1 = spec_add3(W::ent[A1].d1 / 2.f, jt.dmin_base, SPEC_FAR_MARGIN);

  if constexpr (it.kind == VMAS_K_JOINT) {
    V2 qa = pa + rot2(mk(sel(it.ax, jt.ax), sel(it.ay, jt.ay)), ca, sa);
    V2 qb = pb + rot2(mk(sel(it.bx, jt.bx), sel(it.by, jt.by)), cb, sb);
    const float dist = sel(it.dist, jt.dist);
    V2 f_attr = constraint_force(qa, qb, dist, cfg.joint_force, cfg.contact_margin, true);
    V2 f_rep = constraint_force(qa, qb, dist, cfg.joint_force, cfg.contact_margin, false);
    f = f_attr + f_rep;
    V2 fb = neg(f_attr) + neg(f_rep);
    ta = cross2(qa - pa, f);
    tb = cross2(qb - pb, fb);
    if constexpr (!(it.flags & VMAS_IFLAG_JOINT_ROTATE)) {
      float jr = a.joint_rot ? a.joint_rot[(size_t)env * W::N_JOINTS + (o ? I1 : I0)] : sel(it.fixed_rot, jt.fixed_rot);
      float delta = sel(r.rot[A0], r.rot[A1]) - (sel(r.rot[B0], r.rot[B1]) + jr);
      float mag = sqrtf(delta * delta);
      float t = (cfg.torque_constraint_force * sgnf(delta)) * (expf(mag) - 1.f);
      if (mag < 1e-9f) t = 0.f;
      ta = ta + (-t);
      tb = tb + t;
    }
  } else if constexpr (it.kind == VMAS_K_SS) {
    f = constraint_force(pa, pb, dmin, cfg.collision_force, cfg.contact_margin, false);
  } else if constexpr (it.kind == VMAS_K_LS) {  // a = line, b = sphere
    Seg l = seg_a();
    const V2 d = l.p - pb;
    const float lim = sel(LIM_L0, LIM_L1);
    if (!(d.x * d.x + d.y * d.y > lim * lim)) {  // (spec_far_apart)
      V2 cp = closest_point_seg(l, pb);
      V2 f_sphere = constraint_force(pb, cp, dmin, cfg.collision_force, cfg.contact_margin, false);
      f = neg(f_sphere);
      ta = cross2(cp - l.p, f);
    }
  } else if constexpr (it.kind == VMAS_K_LL) {
    Seg l1 = seg_a(), l2 = seg_b();
    if (!spec_far_apart(l1.p, l2.p, l1.half + l2.half + dmin)) {
      Pair c = closest_seg_seg(l1, l2);
      f = constraint_force(c.a, c.b, dmin, cfg.collision_force, cfg.contact_margin, false);
      ta = cross2(c.a - l1.p, f);
      tb = cross2(c.b - l2.p, neg(f));
    }
  } else if constexpr (it.kind == VMAS_K_BS) {  // a = box, b = sphere
    BoxG bx = box_a();
    V2 d0 = pb - bx.p;
    float lx = d0.x * bx.c + d0.y * bx.s, ly = d0.y * bx.c - d0.x * bx.s;
    if (!(fabsf(lx) > sel(LIM_L0, LIM_L1) || fabsf(ly) > sel(LIM_W0, LIM_W1))) {
      V2 cp = closest_point_box(bx, pb);
      V2 inner = cp;
      float d = 0.f;
      if constexpr (!(ea.flags & VMAS_F_HOLLOW)) inner = inner_point_box(pb, cp, bx.p, &d);
      V2 f_sphere = constraint_force(pb, inner, dmin + d, cfg.collision_force, cfg.contact_margin, false);
      f = neg(f_sphere);
      ta = cross2(cp - bx.p, f);
    }
  } else if constexpr (it.kind == VMAS_K_BL) {  // a = box, b = line
    BoxG bx = box_a();
    Seg l = seg_b();
    V2 d0 = l.p - bx.p;
    float lx = d0.x * bx.c + d0.y * bx.s, ly = d0.y * bx.c - d0.x * bx.s;
    float ex = l.half * fabsf(l.c * bx.c + l.s * bx.s), ey = l.half * fabsf(l.s * bx.c - l.c * bx.s);
    if (!(fabsf(lx) - ex > sel(LIM_L0, LIM_L1) || fabsf(ly) - ey > sel(LIM_W0, LIM_W1))) {
      Pair c = closest_box_seg(bx, l);
      V2 inner = c.a;
      float d = 0.f;
      if constexpr (!(ea.flags & VMAS_F_HOLLOW)) inner = inner_point_box(c.b, c.a, bx.p, &d);
      f = constraint_force(inner, c.b, dmin + d, cfg.collision_force, cfg.contact_margin, false);
      ta = cross2(c.a - bx.p, f);
      tb = cross2(c.b - l.p, neg(f));
    }
  } else if constexpr (it.kind == VMAS_K_BB) {
    BoxG b1 = box_a(), b2 = box_b();
    const float circ = sel(W::ent[A0].circ_r + W::ent[B0].circ_r, W::ent[A1].circ_r + W::ent[B1].circ_r);
    if (!spec_far_apart(b1.p, b2.p, circ + dmin)) {
      Pair c = closest_box_box(b1, b2);
      V2 in1 = c.a, in2 = c.b;
      float d1 = 0.f, d2 = 0.f;
      if constexpr (!(ea.flags & VMAS_F_HOLLOW)) in1 = inner_point_box(c.b, c.a, b1.p, &d1);
      if constexpr (!(eb.flags & VMAS_F_HOLLOW)) in2 = inner_point_box(c.a, c.b, b2.p, &d2);
      f = constraint_force(in1, in2, (d1 + d2) + dmin, cfg.collision_force, cfg.contact_margin, false);
      ta = cross2(c.a - b1.p, f);
      tb = cross2(c.b - b2.p, neg(f));
    }
  }
  return ItemOut{f, ta, tb};
}

// false: the broad phase found item I's pair out of range in every env, the item is skipped
template <class W, int I>
DEVI bool spec_item_on(const SpecArgs& a, const uint32_t* mask_words) {
  constexpr int bit = W::item[I].mask_bit;
  if constexpr (bit >= 0) return !a.use_mask || ((mask_words[bit >> 5] >> (bit & 31)) & 1u);
  return true;
}

// item I's contribution into the env's force registers, in the reference's order
template <class W, int I, int E>
DEVI void spec_item_add(EnvRegs<E>& r, const ItemOut& o) {
  constexpr ItemC it = W::item[I];
  constexpr int A = it.a, B = it.b;
  constexpr EntC ea = W::ent[A], eb = W::ent[B];
  if constexpr (ea.flags & VMAS_F_MOVABLE) {
    r.Fx[A] = r.Fx[A] + o.f.x;
    r.Fy[A] = r.Fy[A] + o.f.y;
  }
  if constexpr (ea.flags & VMAS_F_ROTATABLE) r.T[A] = r.T[A] + o.ta;
  if constexpr (eb.flags & VMAS_F_MOVABLE) {
    r.Fx[B] = r.Fx[B] + (-o.f.x);
    r.Fy[B] = r.Fy[B] + (-o.f.y);
  }
  if constexpr (eb.flags & VMAS_F_ROTATABLE) r.T[B] = r.T[B] + o.tb;
}

// One work item evaluated and accumulated by the thread that owns the env.
// TRACK: also record in `sig` whether the item produced a force (env scheduling; off in the default kernel)
template <class W, int I, bool TRACK, int E>
DEVI void spec_item(EnvRegs<E>& r, const SpecArgs& a, long env, const uint32_t* mask_words, uint32_t& sig) {
  if (!spec_item_on<W, I>(a, mask_words)) return;
  const ItemOut o = spec_item_eval<W, I, I>(r, a, env, false);
  if constexpr (TRACK && W::item[I].kind != VMAS_K_JOINT) {
    if (o.f.x != 0.f || o.f.y != 0.f) sig |= 1u << (I & 31);  // this env took the contact branch of item I
  }
  spec_item_add<W, I>(r, o);
}

// ---------------------------------------------------------------------------------------------
// The lane-pair step (step_env_kernel with G = 2): the two lanes 2k, 2k+1 of a warp own one env, both hold its
// whole state.  The work items go in rounds of up to G consecutive items that run the same code; in a round
// each lane evaluates one item, the pair swaps the results with a shuffle and both add every item of the round
// in item order.  Every item reads the state of the substep's start, so the sums are the thread-per-env sums,
// bit for bit.  G = 1: a round is one item, nothing is exchanged: the thread-per-env step.
// ---------------------------------------------------------------------------------------------
template <class W, int G>
struct SpecRounds {
  static_assert(G == 1 || G == 2, "one or two lanes per env");
  struct Table {
    int n;
    int first[W::NI + 1];  // round k: items first[k] .. first[k + 1] - 1
  };
  static constexpr Table make() {
    Table t{};
    int i = 0;
    while (i < W::NI) {
      t.first[t.n++] = i;
      int j = i + 1;
      while (j < W::NI && j - i < G && spec_same_code<W>(i, j)) ++j;
      i = j;
    }
    t.first[t.n] = W::NI;
    return t;
  }
  static constexpr Table table = make();
  static constexpr int N = table.n;
  // the items of round K on the even / odd lane (the same item if the round has only one)
  template <int K>
  static constexpr int I0 = table.first[K];
  template <int K>
  static constexpr int I1 = table.first[K + 1] - 1;
};

// this lane's item of round K (zero if the broad phase skips it)
template <class W, int G, int K, int E>
DEVI ItemOut spec_round_eval(const EnvRegs<E>& r, const SpecArgs& a, long env, const uint32_t* mask_words, bool odd) {
  constexpr int I0 = SpecRounds<W, G>::template I0<K>, I1 = SpecRounds<W, G>::template I1<K>;
  ItemOut o{mk(0.f, 0.f), 0.f, 0.f};
  if (odd ? spec_item_on<W, I1>(a, mask_words) : spec_item_on<W, I0>(a, mask_words))
    o = spec_item_eval<W, I0, I1>(r, a, env, odd);
  return o;
}

// every item of round K into the force registers, in item order: `own` from this lane's spec_round_eval,
// `other` from its partner's
template <class W, int G, int K, int E>
DEVI void spec_round_add(EnvRegs<E>& r, const SpecArgs& a, const uint32_t* mask_words, const ItemOut& own,
                         const ItemOut& other, bool odd) {
  constexpr int I0 = SpecRounds<W, G>::template I0<K>, I1 = SpecRounds<W, G>::template I1<K>;
  if (spec_item_on<W, I0>(a, mask_words)) spec_item_add<W, I0>(r, I0 == I1 || !odd ? own : other);
  if constexpr (I1 != I0) {
    if (spec_item_on<W, I1>(a, mask_words)) spec_item_add<W, I1>(r, odd ? own : other);
  }
}

// the sin / cos evaluations of a substep in spec_trig's order: evaluation k is of entity spec_trig_call(k) / 2,
// of its rotation + pi / 2 if the call is odd (the second axis of a box)
template <class W>
__host__ __device__ constexpr int spec_trig_call(int k) {
  for (int e = 0; e < W::E; ++e) {
    if (!(W::ent[e].flags & VMAS_F_TRIG)) continue;
    if (k-- == 0) return 2 * e;
    if (W::ent[e].shape == VMAS_SHAPE_BOX && k-- == 0) return 2 * e + 1;
  }
  return -1;
}
template <class W>
__host__ __device__ constexpr int spec_n_trig() {
  int n = 0;
  while (spec_trig_call<W>(n) >= 0) ++n;
  return n;
}

// evaluations 2K, 2K + 1 spread over a lane pair (G = 1: evaluation K): this lane's sin / cos
template <class W, int G, int K, int E>
DEVI void spec_trig_round_eval(const EnvRegs<E>& r, bool odd, float& s, float& c) {
  constexpr int C0 = spec_trig_call<W>(G * K), C1 = spec_trig_call<W>(G * K + G - 1 < spec_n_trig<W>() ? G * K + G - 1 : G * K);
  const float x0 = (C0 & 1) ? r.rot[C0 / 2] + SPEC_HALF_PI_F : r.rot[C0 / 2];
  const float x1 = (C1 & 1) ? r.rot[C1 / 2] + SPEC_HALF_PI_F : r.rot[C1 / 2];
  sincosf(C0 != C1 && odd ? x1 : x0, &s, &c);
}
template <class W, int G, int K, int E>
DEVI void spec_trig_round_put(EnvRegs<E>& r, bool odd, float s, float c, float s_other, float c_other) {
  constexpr int C0 = spec_trig_call<W>(G * K), C1 = spec_trig_call<W>(G * K + G - 1 < spec_n_trig<W>() ? G * K + G - 1 : G * K);
  auto put = [&](auto ci, float sv, float cv) {
    constexpr int C = decltype(ci)::value;
    if constexpr (C & 1) {
      r.s2[C / 2] = sv;
      r.c2[C / 2] = cv;
    } else {
      r.s[C / 2] = sv;
      r.c[C / 2] = cv;
    }
  };
  if constexpr (C0 == C1) {
    put(std::integral_constant<int, C0>{}, s, c);
  } else {
    put(std::integral_constant<int, C0>{}, odd ? s_other : s, odd ? c_other : c);
    put(std::integral_constant<int, C1>{}, odd ? s : s_other, odd ? c : c_other);
  }
}

// ---------------------------------------------------------------------------------------------
// per-thread row I/O.  One env's slice of a state tensor ("row", NF floats) is contiguous; the
// owning thread moves it with the widest vector access the row size allows (16 bytes when
// NF % 4 == 0), so a sector is touched by at most two requests instead of once per scalar.
// MASK has one bit per column: vector chunks without any wanted column are skipped at compile
// time; a chunk with at least one is moved whole.
// ---------------------------------------------------------------------------------------------
template <int NF>
struct RowVec {
  static constexpr int W = (NF % 4 == 0) ? 4 : (NF % 2 == 0) ? 2 : 1;
};

__host__ __device__ constexpr uint64_t chunk_closure(uint64_t mask, int nf, int w) {
  uint64_t out = 0;
  for (int c = 0; c < nf; c += w) {
    const uint64_t bits = ((w >= 64 ? ~0ull : ((1ull << w) - 1)) << c);
    if (mask & bits) out |= bits;
  }
  return out;
}

template <int NF, uint64_t MASK>
DEVI void row_load(const float* __restrict__ g, float (&dst)[NF > 0 ? NF : 1]) {
  if constexpr (NF > 0) {
    constexpr int W = RowVec<NF>::W;
    static_for<NF / W>([&](auto ci) {
      constexpr int c = decltype(ci)::value * W;
      if constexpr ((MASK >> c) & ((1ull << W) - 1)) {
        if constexpr (W == 4) {
          const float4 v = *reinterpret_cast<const float4*>(g + c);
          dst[c] = v.x; dst[c + 1] = v.y; dst[c + 2] = v.z; dst[c + 3] = v.w;
        } else if constexpr (W == 2) {
          const float2 v = *reinterpret_cast<const float2*>(g + c);
          dst[c] = v.x; dst[c + 1] = v.y;
        } else {
          dst[c] = g[c];
        }
      }
    });
  }
}

template <int NF, uint64_t MASK>
DEVI void row_store(float* __restrict__ g, const float (&src)[NF > 0 ? NF : 1]) {
  if constexpr (NF > 0) {
    constexpr int W = RowVec<NF>::W;
    static_for<NF / W>([&](auto ci) {
      constexpr int c = decltype(ci)::value * W;
      if constexpr ((MASK >> c) & ((1ull << W) - 1)) {
        if constexpr (W == 4) {
          *reinterpret_cast<float4*>(g + c) = make_float4(src[c], src[c + 1], src[c + 2], src[c + 3]);
        } else if constexpr (W == 2) {
          *reinterpret_cast<float2*>(g + c) = make_float2(src[c], src[c + 1]);
        } else {
          g[c] = src[c];
        }
      }
    });
  }
}

// column masks derived from the world's entity flags at compile time
template <class W>
__host__ __device__ constexpr uint64_t ent_cols(int flag_any, int width) {
  uint64_t m = 0;
  for (int e = 0; e < W::E; ++e)
    if (W::ent[e].flags & flag_any) m |= ((width == 2 ? 3ull : 1ull) << (width * e));
  return m;
}
template <class W>
__host__ __device__ constexpr uint64_t agent_cols(int flag_all, int flag_any, int width) {
  uint64_t m = 0;
  for (int e = 0; e < W::E; ++e) {
    const int f = W::ent[e].flags;
    if ((f & VMAS_F_AGENT) && (f & flag_all) == flag_all && (flag_any == 0 || (f & flag_any)))
      m |= ((width == 2 ? 3ull : 1ull) << (width * W::ent[e].agent));
  }
  return m;
}

// ---------------------------------------------------------------------------------------------
// Per-env physical parameters (domain randomisation).  A world with entities whose mass, friction
// coefficients or gravity are given per env carries `static constexpr int PER_ENV[E]`: the
// VMAS_F_GRAVITY_ENV | VMAS_F_*_ENV bits of each entity.  Every other world has no such member, its
// mask reads zero and not one instruction of its kernels changes.
// ---------------------------------------------------------------------------------------------
template <class W, class = void>
struct SpecPerEnv {
  static constexpr bool any = false;
  __host__ __device__ static constexpr int at(int) { return 0; }
};
template <class W>
struct SpecPerEnv<W, std::void_t<decltype(W::PER_ENV)>> {
  static constexpr bool any = true;
  __host__ __device__ static constexpr int at(int e) { return W::PER_ENV[e]; }
};
template <class W>
__host__ __device__ constexpr bool spec_needs_params() {
  for (int e = 0; e < W::E; ++e)
    if (SpecPerEnv<W>::at(e) & (VMAS_F_MASS_ENV | VMAS_F_LIN_FRIC_ENV | VMAS_F_ANG_FRIC_ENV)) return true;
  return false;
}
template <class W>
__host__ __device__ constexpr bool spec_needs_gravity() {
  for (int e = 0; e < W::E; ++e)
    if (SpecPerEnv<W>::at(e) & VMAS_F_GRAVITY_ENV) return true;
  return false;
}

// One env's per-env parameters, loaded once per launch into registers (only the flagged entries exist after
// unrolling).  The moment of inertia of a per-env mass is rounded as the reference rounds
// `shape.moment_of_inertia(mass)` on a [B, 1] tensor: fp32(fp32(K0 * m) * K1).
template <class W>
struct SpecEnvParams {
  static constexpr int E = W::E;
  float mass[E], inertia[E], lin_fric[E], ang_fric[E], gx[E], gy[E];

  DEVI void load(const SpecArgs& a, const long env) {
    static_for<E>([&](auto ei) {
      constexpr int e = decltype(ei)::value;
      constexpr int m = SpecPerEnv<W>::at(e);
      if constexpr (m & (VMAS_F_MASS_ENV | VMAS_F_LIN_FRIC_ENV | VMAS_F_ANG_FRIC_ENV)) {
        const float4 p = reinterpret_cast<const float4*>(a.ent_params)[(size_t)env * E + e];
        if constexpr (m & VMAS_F_MASS_ENV) {
          mass[e] = p.x;
          inertia[e] = (W::ent[e].inertia_k0 * p.x) * W::ent[e].inertia_k1;
        }
        if constexpr (m & VMAS_F_LIN_FRIC_ENV) lin_fric[e] = p.y;
        if constexpr (m & VMAS_F_ANG_FRIC_ENV) ang_fric[e] = p.z;
      }
      if constexpr (m & VMAS_F_GRAVITY_ENV) {
        const float2 g = reinterpret_cast<const float2*>(a.ent_gravity)[(size_t)env * E + e];
        gx[e] = g.x;
        gy[e] = g.y;
      }
    });
  }
};
static_assert(VMAS_EP_MASS == 0 && VMAS_EP_LIN_FRIC == 1 && VMAS_EP_ANG_FRIC == 2 && VMAS_EP_COLS == 4,
              "SpecEnvParams::load reads an ent_params row as one float4");

// entity e's mass / moment of inertia / friction coefficients: the env's value where the world gives it per env,
// else the compile-time constant
template <class W, int e>
DEVI float spec_mass(const SpecEnvParams<W>* p) {
  if constexpr (SpecPerEnv<W>::at(e) & VMAS_F_MASS_ENV) return p->mass[e];
  else return W::ent[e].mass;
}
template <class W, int e>
DEVI float spec_inertia(const SpecEnvParams<W>* p) {
  if constexpr (SpecPerEnv<W>::at(e) & VMAS_F_MASS_ENV) return p->inertia[e];
  else return W::ent[e].inertia;
}
template <class W, int e>
DEVI float spec_lin_fric(const SpecEnvParams<W>* p) {
  if constexpr (SpecPerEnv<W>::at(e) & VMAS_F_LIN_FRIC_ENV) return p->lin_fric[e];
  else return W::ent[e].lin_fric;
}
template <class W, int e>
DEVI float spec_ang_fric(const SpecEnvParams<W>* p) {
  if constexpr (SpecPerEnv<W>::at(e) & VMAS_F_ANG_FRIC_ENV) return p->ang_fric[e];
  else return W::ent[e].ang_fric;
}

// Tuning knobs.  SPEC_BLOCK: threads (= envs) per block of the specialised kernels.
// SPEC_MIN_BLOCKS: resident blocks per SM the register allocator must leave room for
// (65536 / (SPEC_BLOCK * SPEC_MIN_BLOCKS) registers per thread at most).
#ifndef SPEC_BLOCK
#define SPEC_BLOCK 64
#endif
#ifndef SPEC_MIN_BLOCKS
#define SPEC_MIN_BLOCKS 1
#endif

// ---------------------------------------------------------------------------------------------
// The per-entity statements of one substep, shared by every specialised mapping (thread per env,
// warp tile): same statements, same order => same bits.
// ---------------------------------------------------------------------------------------------
// sin / cos of the entities whose orientation the geometry needs
template <class W, int E>
DEVI void spec_trig(EnvRegs<E>& r) {
  static_for<E>([&](auto ei) {
    constexpr int e = decltype(ei)::value;
    constexpr EntC en = W::ent[e];
    if constexpr (en.flags & VMAS_F_TRIG) {
      sincosf(r.rot[e], &r.s[e], &r.c[e]);
      if constexpr (en.shape == VMAS_SHAPE_BOX) sincosf(r.rot[e] + SPEC_HALF_PI_F, &r.s2[e], &r.c2[e]);
    }
  });
}

// action force / torque (clamped in place), friction, gravity of every entity -> r.Fx, r.Fy, r.T
// (ref core.py:1995-2004, 2018-2102).  `pe`: the env's per-env parameters (worlds with W::PER_ENV only)
template <class W, int E, int NAX>
DEVI void spec_entity_forces(EnvRegs<E>& r, float (&afx)[NAX], float (&afy)[NAX], float (&atq)[NAX],
                             const SpecEnvParams<W>* pe = nullptr) {
  constexpr float sub_dt = W::cfg.sub_dt;
  static_for<E>([&](auto ei) {
    constexpr int e = decltype(ei)::value;
    constexpr EntC en = W::ent[e];
    float Fx = 0.f, Fy = 0.f, T = 0.f;
    if constexpr (en.flags & VMAS_F_AGENT) {
      constexpr int ai = en.agent;
      if constexpr (en.flags & VMAS_F_MOVABLE) {
        if constexpr (en.flags & VMAS_F_MAX_F) {
          const float n = norm2(afx[ai], afy[ai]);
          if (n > en.max_f) {
            afx[ai] = (afx[ai] / n) * en.max_f;
            afy[ai] = (afy[ai] / n) * en.max_f;
          }
        }
        if constexpr (en.flags & VMAS_F_F_RANGE) {
          afx[ai] = clampf(afx[ai], -en.f_range, en.f_range);
          afy[ai] = clampf(afy[ai], -en.f_range, en.f_range);
        }
        Fx = Fx + afx[ai];
        Fy = Fy + afy[ai];
      }
      if constexpr (en.flags & VMAS_F_ROTATABLE) {
        if constexpr (en.flags & VMAS_F_MAX_T) {
          const float n = fabsf(atq[ai]);  // vector_norm of one element
          if (n > en.max_t) atq[ai] = (atq[ai] / n) * en.max_t;
        }
        if constexpr (en.flags & VMAS_F_T_RANGE) atq[ai] = clampf(atq[ai], -en.t_range, en.t_range);
        T = T + atq[ai];
      }
    }
    if constexpr (en.flags & VMAS_F_LIN_FRIC) {
      const float speed = norm2(r.vx[e], r.vy[e]);
      if (speed != 0.f) {
        const float mass = spec_mass<W, e>(pe);
        const float cap = spec_lin_fric<W, e>(pe) * mass;
        Fx = Fx + (-(r.vx[e] / speed)) * fminf(cap, (fabsf(r.vx[e]) / sub_dt) * mass);
        Fy = Fy + (-(r.vy[e] / speed)) * fminf(cap, (fabsf(r.vy[e]) / sub_dt) * mass);
      }
    }
    if constexpr (en.flags & VMAS_F_ANG_FRIC) {
      const float speed = fabsf(r.w[e]);  // vector_norm of one element
      if (speed != 0.f) {
        const float inertia = spec_inertia<W, e>(pe);
        const float cap = spec_ang_fric<W, e>(pe) * inertia;
        T = T + (-(r.w[e] / speed)) * fminf(cap, (fabsf(r.w[e]) / sub_dt) * inertia);
      }
    }
    if constexpr (en.flags & VMAS_F_MOVABLE) {
      const float mass = spec_mass<W, e>(pe);
      if constexpr (W::cfg.has_world_gravity) {
        Fx = Fx + mass * W::cfg.gravity_x;
        Fy = Fy + mass * W::cfg.gravity_y;
      }
      if constexpr (en.flags & VMAS_F_GRAVITY) {
        Fx = Fx + mass * en.grav_x;
        Fy = Fy + mass * en.grav_y;
      }
      if constexpr (SpecPerEnv<W>::at(e) & VMAS_F_GRAVITY_ENV) {
        Fx = Fx + mass * pe->gx[e];
        Fy = Fy + mass * pe->gy[e];
      }
    }
    r.Fx[e] = Fx;
    r.Fy[e] = Fy;
    r.T[e] = T;
  });
}

// semi-implicit Euler of every entity (ref core.py:2862-2908); `sub` is the substep's index in the step
template <class W, int E>
DEVI void spec_integrate(EnvRegs<E>& r, const int sub, const SpecEnvParams<W>* pe = nullptr) {
  constexpr float sub_dt = W::cfg.sub_dt;
  static_for<E>([&](auto ei) {
    constexpr int e = decltype(ei)::value;
    constexpr EntC en = W::ent[e];
    if constexpr (en.flags & VMAS_F_MOVABLE) {
      if (sub == 0) {
        r.vx[e] = r.vx[e] * en.drag_mult;
        r.vy[e] = r.vy[e] * en.drag_mult;
      }
      r.vx[e] = r.vx[e] + div_pos(r.Fx[e], spec_mass<W, e>(pe)) * sub_dt;
      r.vy[e] = r.vy[e] + div_pos(r.Fy[e], spec_mass<W, e>(pe)) * sub_dt;
      if constexpr (en.flags & VMAS_F_MAX_SPEED) {
        const float n = norm2(r.vx[e], r.vy[e]);
        if (n > en.max_speed) {
          r.vx[e] = (r.vx[e] / n) * en.max_speed;
          r.vy[e] = (r.vy[e] / n) * en.max_speed;
        }
      }
      if constexpr (en.flags & VMAS_F_V_RANGE) {
        r.vx[e] = clampf(r.vx[e], -en.v_range, en.v_range);
        r.vy[e] = clampf(r.vy[e], -en.v_range, en.v_range);
      }
      r.px[e] = r.px[e] + r.vx[e] * sub_dt;
      r.py[e] = r.py[e] + r.vy[e] * sub_dt;
      if constexpr (W::cfg.has_x_semidim) r.px[e] = clampf(r.px[e], -W::cfg.x_semidim, W::cfg.x_semidim);
      if constexpr (W::cfg.has_y_semidim) r.py[e] = clampf(r.py[e], -W::cfg.y_semidim, W::cfg.y_semidim);
    }
    if constexpr (en.flags & VMAS_F_ROTATABLE) {
      if (sub == 0) r.w[e] = r.w[e] * en.drag_mult;
      r.w[e] = r.w[e] + div_pos(r.T[e], spec_inertia<W, e>(pe)) * sub_dt;
      r.rot[e] = r.rot[e] + r.w[e] * sub_dt;
    }
  });
}

// The rows of one env (pos, vel, rot, ang_vel, agent force, agent torque) and which vector chunks
// of them are read / written: derived from the world's entity flags at compile time.
// ALL_FORCE: every movable agent's force columns are stored (the whole-step kernel ingests the actions itself);
// F_ACT / T_ACT: the force / torque columns its action prologue writes, stored too (see spec_act_cols)
template <class W, bool ALL_FORCE = false, uint64_t F_ACT = 0, uint64_t T_ACT = 0>
struct SpecRows {
  static constexpr int E = W::E, NA = W::A;
  static constexpr uint64_t ALL_POS = (2 * E >= 64) ? ~0ull : ((1ull << (2 * E)) - 1);
  static constexpr uint64_t MOV2 = ent_cols<W>(VMAS_F_MOVABLE, 2);
  static constexpr uint64_t ROT1 = ent_cols<W>(VMAS_F_ROTATABLE, 1);
  static constexpr uint64_t F_DIRTY =
      (ALL_FORCE ? agent_cols<W>(VMAS_F_MOVABLE, 0, 2) : agent_cols<W>(VMAS_F_MOVABLE, VMAS_F_MAX_F | VMAS_F_F_RANGE, 2)) |
      F_ACT;
  static constexpr uint64_t T_DIRTY = agent_cols<W>(VMAS_F_ROTATABLE, VMAS_F_MAX_T | VMAS_F_T_RANGE, 1) | T_ACT;
  // a vector chunk that will be stored must have been loaded whole (it carries unchanged columns)
  static constexpr uint64_t VEL_IO = chunk_closure(MOV2, 2 * E, RowVec<2 * E>::W);
  static constexpr uint64_t ROT_ST = chunk_closure(ROT1, E, RowVec<E>::W);
  static constexpr uint64_t ROT_LD = ROT_ST | ent_cols<W>(VMAS_F_TRIG | VMAS_F_ROTATABLE, 1);
  static constexpr uint64_t F_ST = chunk_closure(F_DIRTY, 2 * NA, RowVec<2 * NA>::W);
  static constexpr uint64_t T_ST = chunk_closure(T_DIRTY, NA, RowVec<NA>::W);
  static constexpr uint64_t F_LD = F_ST | agent_cols<W>(VMAS_F_MOVABLE, 0, 2);
  static constexpr uint64_t T_LD = T_ST | agent_cols<W>(VMAS_F_ROTATABLE, 0, 1);

  float pos[2 * E], vel[2 * E], rot[E], w[E];
  float f[NA > 0 ? 2 * NA : 1], t[NA > 0 ? NA : 1];

  DEVI void load_pos_rot(const SpecArgs& a, const long env) {
    row_load<2 * E, ALL_POS>(a.st.pos + (size_t)env * 2 * E, pos);
    row_load<E, ROT_LD>(a.st.rot + (size_t)env * E, rot);
  }
  DEVI void load_rest(const SpecArgs& a, const long env) {
    row_load<2 * E, VEL_IO>(a.st.vel + (size_t)env * 2 * E, vel);
    row_load<E, ROT_ST>(a.st.ang_vel + (size_t)env * E, w);
    row_load<2 * NA, F_LD>(a.st.force + (size_t)env * 2 * NA, f);
    row_load<NA, T_LD>(a.st.torque + (size_t)env * NA, t);
  }
  // rows -> registers (pos, rot; trig caches and velocities zeroed)
  DEVI void unpack_pos_rot(EnvRegs<E>& r) const {
    static_for<E>([&](auto ei) {
      constexpr int e = decltype(ei)::value;
      constexpr EntC en = W::ent[e];
      r.px[e] = pos[2 * e];
      r.py[e] = pos[2 * e + 1];
      r.rot[e] = (en.flags & (VMAS_F_TRIG | VMAS_F_ROTATABLE)) ? rot[e] : 0.f;
      r.vx[e] = r.vy[e] = r.w[e] = 0.f;
      r.c[e] = r.s[e] = r.c2[e] = r.s2[e] = 0.f;
    });
  }
  template <int NAX>
  DEVI void unpack_rest(EnvRegs<E>& r, float (&afx)[NAX], float (&afy)[NAX], float (&atq)[NAX]) const {
    static_for<E>([&](auto ei) {
      constexpr int e = decltype(ei)::value;
      constexpr EntC en = W::ent[e];
      if constexpr (en.flags & VMAS_F_MOVABLE) {
        r.vx[e] = vel[2 * e];
        r.vy[e] = vel[2 * e + 1];
      }
      if constexpr (en.flags & VMAS_F_ROTATABLE) r.w[e] = w[e];
      if constexpr (en.flags & VMAS_F_AGENT) {
        if constexpr (en.flags & VMAS_F_MOVABLE) {
          afx[en.agent] = f[2 * en.agent];
          afy[en.agent] = f[2 * en.agent + 1];
        }
        if constexpr (en.flags & VMAS_F_ROTATABLE) atq[en.agent] = t[en.agent];
      }
    });
  }
  // registers -> rows -> global: vector stores of the chunks that hold a changed column.  `lanes` lanes own the
  // env: `lane` stores the rows j = lane (mod lanes) of (pos, vel, rot, ang_vel, force, torque)
  template <int NAX>
  DEVI void store(const SpecArgs& a, const long env, const EnvRegs<E>& r, const float (&afx)[NAX],
                  const float (&afy)[NAX], const float (&atq)[NAX], const int lanes = 1, const int lane = 0) {
    static_for<E>([&](auto ei) {
      constexpr int e = decltype(ei)::value;
      constexpr EntC en = W::ent[e];
      if constexpr (en.flags & VMAS_F_MOVABLE) {
        pos[2 * e] = r.px[e];
        pos[2 * e + 1] = r.py[e];
        vel[2 * e] = r.vx[e];
        vel[2 * e + 1] = r.vy[e];
      }
      if constexpr (en.flags & VMAS_F_ROTATABLE) {
        rot[e] = r.rot[e];
        w[e] = r.w[e];
      }
      if constexpr (en.flags & VMAS_F_AGENT) {
        if constexpr (((en.flags & VMAS_F_MOVABLE) && (ALL_FORCE || (en.flags & (VMAS_F_MAX_F | VMAS_F_F_RANGE)))) ||
                      ((F_ACT >> (2 * en.agent)) & 3ull)) {
          f[2 * en.agent] = afx[en.agent];
          f[2 * en.agent + 1] = afy[en.agent];
        }
        if constexpr (((en.flags & VMAS_F_ROTATABLE) && (en.flags & (VMAS_F_MAX_T | VMAS_F_T_RANGE))) ||
                      ((T_ACT >> en.agent) & 1ull))
          t[en.agent] = atq[en.agent];
      }
    });
    if (lane == 0 % lanes) row_store<2 * E, VEL_IO>(a.st.pos + (size_t)env * 2 * E, pos);
    if (lane == 1 % lanes) row_store<2 * E, VEL_IO>(a.st.vel + (size_t)env * 2 * E, vel);
    if (lane == 2 % lanes) row_store<E, ROT_ST>(a.st.rot + (size_t)env * E, rot);
    if (lane == 3 % lanes) row_store<E, ROT_ST>(a.st.ang_vel + (size_t)env * E, w);
    if (lane == 4 % lanes) row_store<2 * NA, F_ST>(a.st.force + (size_t)env * 2 * NA, f);
    if (lane == 5 % lanes) row_store<NA, T_ST>(a.st.torque + (size_t)env * NA, t);
  }
};

// ---- the whole-step kernel's epilogue -----------------------------------------------------------------
// What Environment.step does after World.step for a scenario written on a StepProgram and an ObservationPlan
// (vmas_b200_post_step: the reward / done glue and the slab-derived observation columns), executed by the
// thread that just stepped the env, on the registers that still hold its state: the program and the column
// table are constexpr members of `P`, every query is resolved against compile-time shapes.  Same functions,
// same arithmetic, same bits as post_step_kernel.

// one element of an env's state after the step: from the registers where the kernel keeps it, else from the slab
template <class W, int FIELD, int OFF>
DEVI float epi_state(const EnvRegs<W::E>& r, const SpecArgs& a, const long env) {
  constexpr int E = W::E;
  if constexpr (FIELD == VMAS_OBS_POS) {
    return (OFF & 1) ? r.py[OFF / 2] : r.px[OFF / 2];
  } else if constexpr (FIELD == VMAS_OBS_VEL) {
    if constexpr (W::ent[OFF / 2].flags & VMAS_F_MOVABLE)
      return (OFF & 1) ? r.vy[OFF / 2] : r.vx[OFF / 2];
    else
      return a.st.vel[(size_t)env * 2 * E + OFF];
  } else if constexpr (FIELD == VMAS_OBS_ROT) {
    if constexpr (W::ent[OFF].flags & (VMAS_F_TRIG | VMAS_F_ROTATABLE))
      return r.rot[OFF];
    else
      return a.st.rot[(size_t)env * E + OFF];
  } else {
    if constexpr (W::ent[OFF].flags & VMAS_F_ROTATABLE)
      return r.w[OFF];
    else
      return a.st.ang_vel[(size_t)env * E + OFF];
  }
}

template <class W, int EI>
DEVI EntG epi_ent(const EnvRegs<W::E>& r, const SpecArgs& a, const long env) {
  constexpr EntC en = W::ent[EI];
  EntG g;
  g.shape = en.shape;
  g.p = mk(r.px[EI], r.py[EI]);
  g.rot = epi_state<W, VMAS_OBS_ROT, EI>(r, a, env);
  g.d0 = en.d0;
  g.d1 = en.d1;
  g.r_plus_lmd = en.r_plus_lmd;
  return g;
}

// The epilogue's per-env inputs (carried shaping terms, loaded flags) are first touched at the very end of the
// thread's instruction chain; requested when the thread starts, their DRAM round trip is over by then.
DEVI void spec_prefetch(const void* p) {
#ifdef __CUDA_ARCH__
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
  (void)p;
#endif
}

template <class P>
DEVI void spec_epilogue_prefetch(const EpiArgs& e, const long env) {
#ifdef __CUDA_ARCH__
  static_for<P::N_PROG>([&](auto ii) {
    constexpr ProgC in = P::prog[decltype(ii)::value];
    if constexpr (in.op == VMAS_OP_SHAPING || in.op == VMAS_OP_LOAD_F32)
      spec_prefetch(static_cast<const float*>(e.buffers[in.a]) + env);
    else if constexpr (in.op == VMAS_OP_LOAD_BOOL)
      spec_prefetch(static_cast<const uint8_t*>(e.buffers[in.a]) + env);
  });
#endif
}

// `lanes` lanes own the env (each holds its whole state and runs the program): `lane` writes the shaping carry
// if it is lane 0, the program's STOREs j = lane (mod lanes) and the observation rows r = lane (mod lanes)
template <class P>
__host__ __device__ constexpr int epi_store_index(int i) {
  int n = 0;
  for (int j = 0; j < i; ++j) n += P::prog[j].op == VMAS_OP_STORE_F32 || P::prog[j].op == VMAS_OP_STORE_BOOL;
  return n;
}

struct EpiOneLane {
  DEVI float operator()(float v) const { return v; }
};

// STEP_COUNT where the counter has been bumped by an earlier launch: a load of it
struct EpiLoadCount {
  DEVI float operator()(const float* steps) const { return *steps; }
};

// P's program reads the step counter (VMAS_OP_STEP_COUNT: a step limit, Environment._limit_program)
template <class P>
__host__ __device__ constexpr bool epi_counts() {
  for (int i = 0; i < P::N_PROG; ++i)
    if (P::prog[i].op == VMAS_OP_STEP_COUNT) return true;
  return false;
}

// from_lane0(v): the value v of lane 0 of the env's lanes (the shaping carry, read by lane 0 only: it overwrites it);
// count(&steps[env]): the env's step counter after this step's increment
template <class W, class P, class X = EpiOneLane, class N = EpiLoadCount>
DEVI void spec_epilogue(const EnvRegs<W::E>& r, const SpecArgs& a, const EpiArgs& e, const long env,
                        const int lanes = 1, const int lane = 0, X from_lane0 = {}, N count = {}) {
  // the step program (ref scenarios/balance.py:197-263 as a StepProgram; see vmas_b200_post_step)
  float pr[VMAS_PROG_REGS];
#pragma unroll
  for (int i = 0; i < VMAS_PROG_REGS; ++i) pr[i] = 0.f;
  static_for<P::N_PROG>([&](auto ii) {
    constexpr ProgC in = P::prog[decltype(ii)::value];
    constexpr int ia = in.arg & 0xFFFF, ib = (in.arg >> 16) & 0xFFFF;
    if constexpr (in.op == VMAS_OP_OVERLAP) {
      pr[in.dst] = pair_overlap(epi_ent<W, ia>(r, a, env), epi_ent<W, ib>(r, a, env)) ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_DISTANCE) {
      pr[in.dst] = pair_distance(epi_ent<W, ia>(r, a, env), epi_ent<W, ib>(r, a, env));
    } else if constexpr (in.op == VMAS_OP_CENTER_DISTANCE) {
      pr[in.dst] = norm2(r.px[ia] - r.px[ib], r.py[ia] - r.py[ib]);
    } else if constexpr (in.op == VMAS_OP_SHAPING) {
      const float d = norm2(r.px[ia] - r.px[ib], r.py[ia] - r.py[ib]);
      const float shaping = d * in.imm;
      float* prev = static_cast<float*>(e.buffers[in.a]) + env;
      float carry = 0.f;
      if (lane == 0) carry = *prev;
      pr[in.dst] = from_lane0(carry) - shaping;
      pr[in.dst + 1] = d;
      if (lane == 0) *prev = shaping;
    } else if constexpr (in.op == VMAS_OP_LOAD_F32) {
      pr[in.dst] = static_cast<const float*>(e.buffers[in.a])[env];
    } else if constexpr (in.op == VMAS_OP_LOAD_BOOL) {
      pr[in.dst] = static_cast<const uint8_t*>(e.buffers[in.a])[env] ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_STEP_COUNT) {
      pr[in.dst] = count(static_cast<const float*>(e.buffers[in.a]) + env);
    } else if constexpr (in.op == VMAS_OP_CONST) {
      pr[in.dst] = in.imm;
    } else if constexpr (in.op == VMAS_OP_ADD) {
      pr[in.dst] = pr[in.a] + pr[in.b];
    } else if constexpr (in.op == VMAS_OP_SUB) {
      pr[in.dst] = pr[in.a] - pr[in.b];
    } else if constexpr (in.op == VMAS_OP_MUL) {
      pr[in.dst] = pr[in.a] * pr[in.b];
    } else if constexpr (in.op == VMAS_OP_MIN) {
      pr[in.dst] = fminf(pr[in.a], pr[in.b]);
    } else if constexpr (in.op == VMAS_OP_MAX) {
      pr[in.dst] = fmaxf(pr[in.a], pr[in.b]);
    } else if constexpr (in.op == VMAS_OP_NEG) {
      pr[in.dst] = -pr[in.a];
    } else if constexpr (in.op == VMAS_OP_OR) {
      pr[in.dst] = (pr[in.a] != 0.f || pr[in.b] != 0.f) ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_AND) {
      pr[in.dst] = (pr[in.a] != 0.f && pr[in.b] != 0.f) ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_NOT) {
      pr[in.dst] = pr[in.a] != 0.f ? 0.f : 1.f;
    } else if constexpr (in.op == VMAS_OP_LT) {
      pr[in.dst] = pr[in.a] < pr[in.b] ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_LE) {
      pr[in.dst] = pr[in.a] <= pr[in.b] ? 1.f : 0.f;
    } else if constexpr (in.op == VMAS_OP_WHERE) {
      pr[in.dst] = pr[in.a] != 0.f ? pr[in.b] : pr[in.arg & 0xFF];
    } else if constexpr (in.op == VMAS_OP_STORE_F32) {
      if (lane == epi_store_index<P>(decltype(ii)::value) % lanes) static_cast<float*>(e.buffers[in.b])[env] = pr[in.a];
    } else if constexpr (in.op == VMAS_OP_STORE_BOOL) {
      if (lane == epi_store_index<P>(decltype(ii)::value) % lanes)
        static_cast<uint8_t*>(e.buffers[in.b])[env] = pr[in.a] != 0.f ? 1 : 0;
    }
  });
  // the observation rows (ref scenarios/balance.py:236-262 as an ObservationPlan): [rows, B, width] of
  // P::OBS_DTYPE.  16-bit rows are rounded here, in registers, pair by pair as the values come, and stored as one
  // 4-byte word per pair: 8-byte stores of 4 columns cost the lane-pair kernel of balance a register (127, not 126)
  if constexpr (P::OBS_ROWS > 0) {
    constexpr int DT = P::OBS_DTYPE, F = P::OBS_WIDTH;
    constexpr int VEC = DT != VMAS_DTYPE_F32 ? (F % 2 == 0 ? 2 : 1) : F % 4 == 0 ? 4 : 1;
    static_for<P::OBS_ROWS>([&](auto ri) {
      constexpr int row = decltype(ri)::value;
      if (lane != row % lanes) return;
      const size_t at = ((size_t)row * a.batch_dim + env) * F;
      float* dst = static_cast<float*>(e.obs_out) + at;
      uint16_t* dst16 = static_cast<uint16_t*>(e.obs_out) + at;
      static_for<F / VEC>([&](auto gi) {
        constexpr int c0 = decltype(gi)::value * VEC;
        float v[VEC];
        [[maybe_unused]] uint32_t packed[VEC / 2 > 0 ? VEC / 2 : 1];
        bool all = true;
        static_for<VEC>([&](auto ki) {
          constexpr int k = decltype(ki)::value;
          constexpr ObsColC col = P::obs[row * F + c0 + k];
          v[k] = 0.f;
          if constexpr (col.op == VMAS_OBS_REG) {
            v[k] = pr[col.src];  // a value the step program (above, same thread) computed
          } else if constexpr (col.op != VMAS_OBS_SKIP) {
            v[k] = epi_state<W, (col.src >> 24) & 3, col.src & 0xFFFFFF>(r, a, env);
            if constexpr (col.op == VMAS_OBS_DIFF)
              v[k] = v[k] - epi_state<W, (col.src2 >> 24) & 3, col.src2 & 0xFFFFFF>(r, a, env);
            if constexpr (col.op == VMAS_OBS_REMAINDER) v[k] = obs_remainder(v[k], col.par);
          } else {
            all = false;
          }
          if constexpr (DT != VMAS_DTYPE_F32 && k % 2 == 1) packed[k / 2] = obs16x2_bits<DT>(v[k - 1], v[k]);
        });
        if constexpr (DT == VMAS_DTYPE_F32) {
          if constexpr (VEC == 4) {
            if (all) {
              *reinterpret_cast<float4*>(dst + c0) = make_float4(v[0], v[1], v[2], v[3]);
              return;
            }
          }
        } else if constexpr (VEC == 2) {
          if (all) {
            *reinterpret_cast<uint32_t*>(dst16 + c0) = packed[0];
            return;
          }
        }
        static_for<VEC>([&](auto ki) {
          constexpr int k = decltype(ki)::value;
          if constexpr (P::obs[row * F + c0 + k].op != VMAS_OBS_SKIP) {
            if constexpr (DT == VMAS_DTYPE_F32) dst[c0 + k] = v[k];
            else dst16[c0 + k] = obs16_bits<DT>(v[k]);
          }
        });
      });
    });
  }
}

// ---- the LIDAR stage of the epilogue --------------------------------------------------------------------------------
// What cast_rays_batched_kernel does behind the observation launch of a plan with LIDAR terms, on the registers that
// hold the env's state after the last substep: every ray of every sensor of P (P::N_LIDAR; a plan without LIDAR terms
// has no such member and no code here), its reading stored into the sensor's columns of the observation rows.  Same
// functions (rays.cuh), same targets in the same order, same reach test, same fp32(angle + rot) and sincosf, same
// max_range - distance: the same bits.
template <class P, class = void>
struct EpiLidars {
  static constexpr int N = 0;
};
template <class P>
struct EpiLidars<P, std::void_t<decltype(P::N_LIDAR)>> {
  static constexpr int N = P::N_LIDAR;
};

// target T of a sensor as the epilogue holds it: position in the registers, heading from epi_state, shape constants
template <class W, int T>
struct EpiRayTarget {
  const EnvRegs<W::E>& r;
  const SpecArgs& a;
  long env;
  DEVI int shape() const { return W::ent[T].shape; }
  DEVI V2 pos() const { return mk(r.px[T], r.py[T]); }
  DEVI float rot() const { return epi_state<W, VMAS_OBS_ROT, T>(r, a, env); }
  DEVI float d0() const { return W::ent[T].d0; }
  DEVI float d1() const { return W::ent[T].d1; }
};

// G lanes own the env: ray k of a sensor goes to lane k % G, which stores its column.  The rays of a sensor are a loop
// (not unrolled: a sensor's target tests are emitted once, not once per ray, so that the kernel's code stays within
// what the instruction caches hold); a ray's angle is picked from the compile-time table by its index.
template <class W, class P, int G>
DEVI void spec_lidar(const EnvRegs<W::E>& r, const SpecArgs& a, const EpiArgs& e, const long env, const bool odd) {
  if constexpr (EpiLidars<P>::N > 0) {
    constexpr int R = P::LIDAR_RAYS, F = P::OBS_WIDTH, DT = P::OBS_DTYPE;
    static_for<P::N_LIDAR>([&](auto qi) {
      using Q = decltype(qi);
      constexpr LidarC L = P::lidar[Q::value];
      const V2 o = mk(r.px[L.src], r.py[L.src]);
      const float src_rot = epi_state<W, VMAS_OBS_ROT, L.src>(r, a, env);
      // the exact early-out of the batched kernel's phase A: a bit per target within the sensor's reach
      uint32_t reach = 0u;
      static_for<L.n_targets>([&](auto ti) {
        constexpr int t = P::lidar[Q::value].target[decltype(ti)::value];
        if (ray_in_reach(o, mk(r.px[t], r.py[t]), W::ent[t].circ_r, P::lidar[Q::value].max_range))
          reach |= 1u << decltype(ti)::value;
      });
      const size_t at = ((size_t)L.row * a.batch_dim + env) * F + L.col;
#pragma unroll 1
      for (int k = G > 1 && odd ? 1 : 0; k < R; k += G) {
        float d = L.max_range;
        if (reach) {
          float angle = 0.f;
          static_for<R>([&](auto ki) {
            constexpr float value = P::lidar_angle[Q::value * R + decltype(ki)::value];
            if (k == decltype(ki)::value) angle = value;
          });
          float ds, dc;
          sincosf(angle + src_rot, &ds, &dc);
          static_for<L.n_targets>([&](auto ti) {
            constexpr int t = P::lidar[Q::value].target[decltype(ti)::value];
            if ((reach >> decltype(ti)::value) & 1u)
              d = tmin(d, ray_vs_shape(EpiRayTarget<W, t>{r, a, env}, o, dc, ds, P::lidar[Q::value].max_range));
          });
        }
        const float v = P::LIDAR_FLIP ? L.max_range - d : d;
        if constexpr (DT == VMAS_DTYPE_F32) static_cast<float*>(e.obs_out)[at + k] = v;
        else static_cast<uint16_t*>(e.obs_out)[at + k] = obs16_bits<DT>(v);
      }
    });
  }
}

// One env, all of `a.n_substeps` substeps, state in the calling thread's registers.  `P` (not void): the
// step's epilogue runs behind the last substep (the whole-step kernel).
template <class W, bool TRACK = false, class P = void>
DEVI void spec_env_step(const SpecArgs& a, const long env, const uint32_t (&mask_words)[W::MASK_WORDS > 0 ? W::MASK_WORDS : 1],
                        const EpiArgs* epi = nullptr) {
  constexpr int E = W::E, NA = W::A, NI = W::NI;
  if (env >= a.batch_dim) return;
  SpecRows<W> rows;
  rows.load_pos_rot(a, env);
  rows.load_rest(a, env);
  if constexpr (!std::is_void_v<P>) {
    if (a.first_substep + a.n_substeps == W::cfg.substeps) spec_epilogue_prefetch<P>(*epi, env);
  }
  EnvRegs<E> r;
  float afx[NA > 0 ? NA : 1], afy[NA > 0 ? NA : 1], atq[NA > 0 ? NA : 1];
  rows.unpack_pos_rot(r);
  rows.unpack_rest(r, afx, afy, atq);
  SpecEnvParams<W> pe;
  if constexpr (SpecPerEnv<W>::any) pe.load(a, env);
  uint32_t sig = 0;
  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    spec_trig<W>(r);
    spec_entity_forces<W>(r, afx, afy, atq, &pe);
    // joints and contacts, in accumulation order
    static_for<NI>([&](auto ii) { spec_item<W, decltype(ii)::value, TRACK>(r, a, env, mask_words, sig); });
    spec_integrate<W>(r, sub, &pe);
  }
  rows.store(a, env, r, afx, afy, atq);
  if constexpr (!std::is_void_v<P>) {
    if (a.first_substep + a.n_substeps == W::cfg.substeps) {
      spec_epilogue<W, P>(r, a, *epi, env);
      spec_lidar<W, P, 1>(r, a, *epi, env, false);
    }
  }
  if constexpr (TRACK) {
    if (a.sig) a.sig[env] = (a.first_substep == 0 ? 0u : a.sig[env]) | sig;  // OR over the substeps of a step
  }
}

// ---- the action prologue of the one-kernel step (step_env_kernel), one lane at a time ----------------------------
// Round J of G lanes per env: agent k0 = G J on the even lane, k1 = G J + G - 1 on the odd lane (k1 = k0 for a lone
// agent or G = 1: both lanes decode it).
template <class P, int G, int J>
struct SpecActRound {
  static constexpr int k0 = J * G, k1 = k0 + G - 1 < P::N_ACT ? k0 + G - 1 : k0;
};

// The lane's agent's action, decoded as the ingest kernel does (ingest_continuous / ingest_discrete; a discrete
// flat index is unravelled by the same truncating / and %), stored to agent.action.u (live envs; a lone agent's
// from the even lane) and returned.  `bad` collects the flag.  No clamp for discrete kinds.
template <class P, int G, int J>
DEVI float2 spec_ingest_lane(const ActArgs& act, const long env, const bool odd, const bool live, bool& bad) {
  constexpr int k0 = SpecActRound<P, G, J>::k0, k1 = SpecActRound<P, G, J>::k1;
  constexpr ActC c0 = P::act[k0], c1 = P::act[k1];
  static_assert(c0.kind == c1.kind, "one action kind per round");
  const bool o = k0 != k1 && odd;
  const float range0 = o ? c1.range0 : c0.range0, range1 = o ? c1.range1 : c0.range1;
  float2 u;
  if constexpr (c0.kind == VMAS_ACT_CONTINUOUS) {
    const float2 v = reinterpret_cast<const float2*>(o ? act.actions[k1] : act.actions[k0])[env];
    const float ux = ingest_continuous(v.x, range0, o ? c1.mult0 : c0.mult0, act.clamp, bad);
    u = make_float2(ux, ingest_continuous(v.y, range1, o ? c1.mult1 : c0.mult1, act.clamp, bad));
  } else {
    const void* in = o ? act.actions[k1] : act.actions[k0];
    const long long n1 = o ? c1.n1 : c0.n1;
    long long i0, i1;
    if constexpr (c0.kind == VMAS_ACT_DISCRETE) {  // [B, 1]: the flat index of the product of the two components
      const long long flat = static_cast<const long long*>(in)[env];
      i0 = flat / n1;
      i1 = flat % n1;
    } else {  // [B, 2]
      const ActIdx2 k = static_cast<const ActIdx2*>(in)[env];
      i0 = k.i0;
      i1 = k.i1;
    }
    const float ux = ingest_discrete(i0, o ? c1.n0 : c0.n0, range0, o ? c1.mult0 : c0.mult0, bad);
    u = make_float2(ux, ingest_discrete(i1, n1, range1, o ? c1.mult1 : c0.mult1, bad));
  }
  if (live && (k0 != k1 || !odd)) reinterpret_cast<float2*>(o ? act.u[k1] : act.u[k0])[env] = u;
  return u;
}

// ... and round J's force rows on the lane: its own u, and p = the partner lane's u (a pair of agents only)
template <class P, int G, int J>
DEVI void spec_ingest_put(const float2 u, const float2 p, const bool odd, float* afx, float* afy) {
  constexpr int k0 = SpecActRound<P, G, J>::k0, k1 = SpecActRound<P, G, J>::k1;
  constexpr ActC c0 = P::act[k0], c1 = P::act[k1];
  if constexpr (k0 == k1) {
    afx[c0.agent] = u.x;
    afy[c0.agent] = u.y;
  } else {
    afx[c0.agent] = odd ? p.x : u.x;
    afy[c0.agent] = odd ? p.y : u.y;
    afx[c1.agent] = odd ? u.x : p.x;
    afy[c1.agent] = odd ? u.y : p.y;
  }
}

// ---- the prologue's rounds with other action models (any round with an agent that is not holonomic with 2
// components).  Each lane runs its own agent's decode and model under a branch on the lane: the agents of a pair may
// differ in model and action kind.  A lane hands its partner the force and the torque it computed.
struct ActBody {  // the state an action model reads: the agent's heading, angular velocity and velocity
  float rot, w;
  float2 vel;
};
struct ActOut {  // what it returns: the force and torque rows
  float2 f;
  float t;
};

// the force / torque columns (width 2 / 1) that the prologue of P writes
template <class P>
__host__ __device__ constexpr uint64_t spec_act_cols(bool torque) {
  uint64_t m = 0;
  for (int k = 0; k < P::N_ACT; ++k) {
    const ActC& c = P::act[k];
    if (torque ? dyn_writes_torque(c.dyn) : dyn_writes_force(c.dyn)) m |= (torque ? 1ull : 3ull) << ((torque ? 1 : 2) * c.agent);
  }
  return m;
}
// round J runs spec_ingest_lane (both agents holonomic with 2 components and of one kind), else spec_act_lane
template <class P, int G, int J>
__host__ __device__ constexpr bool spec_act_lean() {
  constexpr ActC c0 = P::act[SpecActRound<P, G, J>::k0], c1 = P::act[SpecActRound<P, G, J>::k1];
  return act_holonomic2(c0) && act_holonomic2(c1) && c0.kind == c1.kind;
}

// Agent k's action: decoded as ingest_actions_body decodes it (the same helpers, the same unravel order), through
// its model (act_model, the ingest kernel's device functions).  u is stored to agent.action.u if `store_u`.
// `body(std::integral_constant<int, k>{})`: the agent's ActBody (read only by the models that need it).
template <class P, int k, class Body>
DEVI ActOut spec_act_agent(const ActArgs& act, const long env, const bool store_u, bool& bad, Body&& body) {
  constexpr ActC c = P::act[k];
  constexpr int sz = c.size;
  float u[VMAS_MAX_ACTION_SIZE];
  if constexpr (c.kind == VMAS_ACT_CONTINUOUS) {
    const float* in = act.actions[k] + (size_t)env * sz;
    static_for<sz>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      u[j] = ingest_continuous(in[j], act_range(c, j), act_mult(c, j), act.clamp, bad);
    });
  } else {
    const long long* idx_in = reinterpret_cast<const long long*>(act.actions[k]);
    long long flat = c.kind == VMAS_ACT_DISCRETE ? idx_in[env] : 0;
    static_for<sz>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      constexpr ActC c = P::act[k];  // (the enclosing one is not a constant in here)
      long long i;
      if constexpr (c.kind == VMAS_ACT_DISCRETE) {  // unravel the flat index of the cartesian product
        long long stride = 1;
        for (int m = j + 1; m < sz; ++m) stride *= act_n(c, m);
        i = flat / stride;
        flat = flat % stride;
      } else {
        i = idx_in[(size_t)env * sz + j];
      }
      u[j] = ingest_discrete(i, act_n(c, j), act_range(c, j), act_mult(c, j), bad);
    });
  }
  ActOut o;
  o.f = make_float2(0.f, 0.f);
  o.t = 0.f;
  if constexpr (c.dyn == VMAS_DYN_HOLONOMIC || c.dyn == VMAS_DYN_HOLONOMIC_ROT) {
    o.f = make_float2(u[0], u[1]);
    if constexpr (c.dyn == VMAS_DYN_HOLONOMIC_ROT) o.t = u[2];
  } else if constexpr (c.dyn == VMAS_DYN_FORWARD) {
    o.f = forward_force(u[0], body(std::integral_constant<int, k>{}).rot);
  } else if constexpr (c.dyn == VMAS_DYN_ROTATION) {
    o.t = u[0];
  } else {
    static_assert(c.dyn == VMAS_DYN_DIFF_DRIVE, "an action model the prologue has not (codegen.PROLOGUE_MODELS)");
    const ActBody b = body(std::integral_constant<int, k>{});
    const float dt = c.params[0], mass = c.params[1], inertia = c.params[2];
    constexpr bool rk4 = c.params[3] != 0.f;
    const Pose3 d = diff_drive_pose(u[0], u[1], b.rot, dt, rk4);
    o.f = kinematic_force(d, dt, mass, inertia, b.vel, b.w, o.t);
  }
  if (store_u) {
    static_for<sz>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      act.u[k][(size_t)env * sz + j] = u[j];
    });
  }
  return o;
}

// The lane's agent of round J (k1 on the odd lane of a pair, else k0; a lone agent: both lanes, the even one stores)
template <class P, int G, int J, class Body>
DEVI ActOut spec_act_lane(const ActArgs& act, const long env, const bool odd, const bool live, bool& bad, Body&& body) {
  constexpr int k0 = SpecActRound<P, G, J>::k0, k1 = SpecActRound<P, G, J>::k1;
  if constexpr (k0 == k1) {
    return spec_act_agent<P, k0>(act, env, live && !odd, bad, body);
  } else {
    if (odd) return spec_act_agent<P, k1>(act, env, live, bad, body);
    return spec_act_agent<P, k0>(act, env, live, bad, body);
  }
}

// ... and round J's rows on the lane: own = its result, p = the partner lane's (a pair of agents only).  Only the
// rows each model writes.
template <class P, int G, int J>
DEVI void spec_act_put(const ActOut& own, const ActOut& p, const bool odd, float* afx, float* afy, float* atq) {
  constexpr int k0 = SpecActRound<P, G, J>::k0, k1 = SpecActRound<P, G, J>::k1;
  constexpr ActC c0 = P::act[k0], c1 = P::act[k1];
  const ActOut& r0 = k0 == k1 || !odd ? own : p;
  if constexpr (dyn_writes_force(c0.dyn)) {
    afx[c0.agent] = r0.f.x;
    afy[c0.agent] = r0.f.y;
  }
  if constexpr (dyn_writes_torque(c0.dyn)) atq[c0.agent] = r0.t;
  if constexpr (k0 != k1) {
    const ActOut& r1 = odd ? own : p;
    if constexpr (dyn_writes_force(c1.dyn)) {
      afx[c1.agent] = r1.f.x;
      afy[c1.agent] = r1.f.y;
    }
    if constexpr (dyn_writes_torque(c1.dyn)) atq[c1.agent] = r1.t;
  }
}

#ifdef __CUDACC__
// SCHED: the env-scheduling variant (thread t steps env order[t], signatures recorded); the default
// kernel carries none of that code
template <class W, bool SCHED = false>
__global__ void __launch_bounds__(W::BLOCK, W::MIN_BLOCKS) step_spec_kernel(const SpecArgs a) {
  constexpr int MW = W::MASK_WORDS;
  const long tid = (long)blockIdx.x * W::BLOCK + threadIdx.x;

  // the block's copy of the broad-phase mask (ref core.py:2797-2801); the last block to have copied
  // it clears it for the next substep (no memset node: CUDA-graph safe)
  uint32_t mask_words[MW > 0 ? MW : 1];
  if constexpr (MW > 0) {
    __shared__ uint32_t s_mask[MW];
    if (a.use_mask) {
      for (int w = threadIdx.x; w < MW; w += W::BLOCK) s_mask[w] = a.mask[w];
      __syncthreads();
      if (threadIdx.x == 0) {
        __threadfence();
        unsigned done = atomicAdd(&a.mask[MW], 1u);
        if (done == gridDim.x - 1) {
          for (int w = 0; w < MW; ++w) a.mask[w] = 0u;
          a.mask[MW] = 0u;
        }
      }
#pragma unroll
      for (int w = 0; w < MW; ++w) mask_words[w] = s_mask[w];
    }
  }
  if (tid >= a.batch_dim) return;
  if constexpr (SCHED) {
    // env scheduling: with an order table, neighbouring threads step envs with the same contact pattern
    const long env = a.order ? (long)a.order[tid] : tid;
    spec_env_step<W, true>(a, env, mask_words);
  } else {
    spec_env_step<W, false>(a, tid, mask_words);
  }
}

// The whole-step kernel: step_spec_kernel with the epilogue P behind the last substep.
template <class W, class P>
__global__ void __launch_bounds__(W::BLOCK, W::MIN_BLOCKS) step_fused_kernel(const SpecArgs a, const EpiArgs e) {
  static_assert(!SpecPerEnv<W>::any, "no whole-step kernel for worlds with per-env parameters");
  constexpr int MW = W::MASK_WORDS;
  const long tid = (long)blockIdx.x * W::BLOCK + threadIdx.x;
  uint32_t mask_words[MW > 0 ? MW : 1];
  if constexpr (MW > 0) {
    __shared__ uint32_t s_mask[MW];
    if (a.use_mask) {
      for (int w = threadIdx.x; w < MW; w += W::BLOCK) s_mask[w] = a.mask[w];
      __syncthreads();
      if (threadIdx.x == 0) {
        __threadfence();
        unsigned done = atomicAdd(&a.mask[MW], 1u);
        if (done == gridDim.x - 1) {
          for (int w = 0; w < MW; ++w) a.mask[w] = 0u;
          a.mask[MW] = 0u;
        }
      }
#pragma unroll
      for (int w = 0; w < MW; ++w) mask_words[w] = s_mask[w];
    }
  }
  if (tid >= a.batch_dim) return;
  spec_env_step<W, false, P>(a, tid, mask_words, &e);
}

// ---- the whole Environment.step as ONE kernel -----------------------------------------------------------
// step_fused_kernel plus what the ingest launch in front of it does (vmas_b200_ingest_actions_broad_phase):
// every thread decodes its env's actions (continuous, discrete or multi-discrete: ref environment.py:616-707; through
// each agent's action model, ref dynamics/*.py) straight into the force / torque registers, counts the step, and tests its env's
// masked pairs for the batch-wide broad phase (ref core.py:2797-2801); the mask is complete once every block
// has contributed — a grid-wide barrier, which needs all blocks resident (cooperative launch; the launcher
// says no for batches beyond that and the caller keeps the separate ingest launch).
//   a.mask: per substep [MASK_WORDS] bits, [MASK_WORDS] arrivals at the barrier, [MASK_WORDS + 1] unused but for
//   substep 0's, which counts the blocks done with every mask (substeps x (MASK_WORDS + 2) words, zero between
//   launches)
template <class W>
__host__ __device__ constexpr int spec_first_masked() {
  for (int i = 0; i < W::NI; ++i)
    if (W::item[i].mask_bit >= 0) return i;
  return W::NI;
}

// word w of the mask with every masked item's bit set: the most the batch-wide OR can hold
template <class W>
__host__ __device__ constexpr uint32_t spec_mask_full(int w) {
  uint32_t m = 0u;
  for (int i = 0; i < W::NI; ++i)
    if (W::item[i].mask_bit >= 0 && (W::item[i].mask_bit >> 5) == w) m |= 1u << (W::item[i].mask_bit & 31);
  return m;
}

DEVI unsigned ld_acquire_u32(const uint32_t* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// fire-and-forget: nothing comes back to wait on
DEVI void red_or_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.relaxed.gpu.global.or.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// the release orders this thread's earlier stores and reductions (the mask bits) before the add
DEVI void red_release_add_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
DEVI unsigned atom_acq_rel_add_u32(uint32_t* p, uint32_t v) {
  unsigned old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// the k-th masked work item, in item order
template <class W>
__host__ __device__ constexpr int spec_masked_item(int k) {
  for (int i = 0; i < W::NI; ++i)
    if (W::item[i].mask_bit >= 0 && k-- == 0) return i;
  return -1;
}
template <class W>
__host__ __device__ constexpr int spec_n_masked() {
  int n = 0;
  for (int i = 0; i < W::NI; ++i) n += W::item[i].mask_bit >= 0;
  return n;
}

// the entity of agent row `agent`
template <class W>
__host__ __device__ constexpr int spec_agent_entity(int agent) {
  for (int e = 0; e < W::E; ++e)
    if ((W::ent[e].flags & VMAS_F_AGENT) && W::ent[e].agent == agent) return e;
  return -1;
}

// the partner lane's value (lanes 2k, 2k + 1)
DEVI float pair_swap(float v) { return __shfl_xor_sync(0xffffffffu, v, 1); }

// what the partner lane evaluated in round K (only the parts some item of the round adds somewhere)
template <class W, int G, int K>
DEVI ItemOut spec_round_swap(const ItemOut& o) {
  constexpr int I0 = SpecRounds<W, G>::template I0<K>, I1 = SpecRounds<W, G>::template I1<K>;
  if constexpr (I0 == I1) {
    return o;
  } else {
    constexpr int fa = W::ent[W::item[I0].a].flags | W::ent[W::item[I1].a].flags;
    constexpr int fb = W::ent[W::item[I0].b].flags | W::ent[W::item[I1].b].flags;
    ItemOut p = o;
    if constexpr ((fa | fb) & VMAS_F_MOVABLE) {
      p.f.x = pair_swap(o.f.x);
      p.f.y = pair_swap(o.f.y);
    }
    if constexpr (fa & VMAS_F_ROTATABLE) p.ta = pair_swap(o.ta);
    if constexpr (fb & VMAS_F_ROTATABLE) p.tb = pair_swap(o.tb);
    return p;
  }
}

// G lanes per env (see SpecRounds): lanes 2k, 2k + 1 of a warp own one env, a block holds W::BLOCK envs whatever
// G.  Both lanes load the env's rows (the same addresses: no extra bytes) and keep its whole state; they split
// the action ingest, the broad-phase tests, the sin / cos evaluations, the work items, the row stores, the
// program's stores and the observation rows, and exchange what the other lane needs by shuffles.
template <class W, class P, int G>
__global__ void __launch_bounds__(W::BLOCK* G, (W::MIN_BLOCKS / G > 0 ? W::MIN_BLOCKS / G : 1))
    step_env_kernel(const SpecArgs a, const EpiArgs e, const ActArgs act) {
  static_assert(!SpecPerEnv<W>::any, "no whole-step kernel for worlds with per-env parameters");
  constexpr int MW = W::MASK_WORDS, E = W::E, NA = W::A;
  using R = SpecRounds<W, G>;
  const long tid = ((long)blockIdx.x * (W::BLOCK * G) + threadIdx.x) / G;
  const bool odd = G > 1 && (threadIdx.x & 1);
  const bool live = tid < a.batch_dim;
  const long env = live ? tid : (long)a.batch_dim - 1;  // (the tail threads shadow the last env and store nothing)
  SpecRows<W, true, spec_act_cols<P>(false), spec_act_cols<P>(true)> rows;
  rows.load_pos_rot(a, env);
  rows.load_rest(a, env);
  spec_epilogue_prefetch<P>(e, env);
#ifdef __CUDA_ARCH__
  if (act.steps) spec_prefetch(act.steps + env);
#endif
  EnvRegs<E> r;
  float afx[NA > 0 ? NA : 1], afy[NA > 0 ? NA : 1], atq[NA > 0 ? NA : 1];
  rows.unpack_pos_rot(r);
  rows.unpack_rest(r, afx, afy, atq);
  // the actions: agents k0 = G j and k1 = G j + G - 1 on the lanes of a pair
  bool bad = false;
  static_for<(P::N_ACT + G - 1) / G>([&](auto ji) {
    constexpr int J = decltype(ji)::value;
    constexpr int k0 = SpecActRound<P, G, J>::k0, k1 = SpecActRound<P, G, J>::k1;
    if constexpr (spec_act_lean<P, G, J>()) {
      const float2 u = spec_ingest_lane<P, G, J>(act, env, odd, live, bad);
      if constexpr (k0 == k1)
        spec_ingest_put<P, G, J>(u, u, odd, afx, afy);
      else
        spec_ingest_put<P, G, J>(u, make_float2(pair_swap(u.x), pair_swap(u.y)), odd, afx, afy);
    } else {
      // the models read the agent's state from the registers loaded above (nothing has moved yet); an entity whose
      // heading or velocities the substeps do not use has them in the slab only
      auto body = [&](auto ki) {
        constexpr int ent = spec_agent_entity<W>(P::act[decltype(ki)::value].agent);
        constexpr int f = W::ent[ent].flags;
        const size_t at = (size_t)env * E + ent;
        ActBody b;
        if constexpr (f & (VMAS_F_TRIG | VMAS_F_ROTATABLE)) b.rot = r.rot[ent];
        else b.rot = a.st.rot[at];
        if constexpr (f & VMAS_F_ROTATABLE) b.w = r.w[ent];
        else b.w = a.st.ang_vel[at];
        if constexpr (f & VMAS_F_MOVABLE) b.vel = make_float2(r.vx[ent], r.vy[ent]);
        else b.vel = reinterpret_cast<const float2*>(a.st.vel)[at];
        return b;
      };
      const ActOut own = spec_act_lane<P, G, J>(act, env, odd, live, bad, body);
      ActOut p = own;
      if constexpr (k0 != k1) {
        constexpr ActC c0 = P::act[k0], c1 = P::act[k1];
        if constexpr (dyn_writes_force(c0.dyn) || dyn_writes_force(c1.dyn)) p.f = make_float2(pair_swap(own.f.x), pair_swap(own.f.y));
        if constexpr (dyn_writes_torque(c0.dyn) || dyn_writes_torque(c1.dyn)) p.t = pair_swap(own.t);
      }
      spec_act_put<P, G, J>(own, p, odd, afx, afy, atq);
    }
  });
  if constexpr (G > 1) bad = __shfl_xor_sync(0xffffffffu, (int)bad, 1) || bad;
  // a program that reads the step counter gets the sum from here: a reload in the epilogue would race the even
  // lane's store on the odd lane (launch_env refuses such a kernel without a counter)
  [[maybe_unused]] float count = 0.f;
  if constexpr (epi_counts<P>()) {
    if (live && !odd) {
      if (bad && act.bad_flag) *act.bad_flag = 1;
      count = act.steps[env] + 1.f;
      act.steps[env] = count;
    }
    if constexpr (G > 1) {
      const float even = pair_swap(count);
      if (odd) count = even;
    }
  } else {
    if (live && !odd) {
      if (bad && act.bad_flag) *act.bad_flag = 1;
      if (act.steps) act.steps[env] = act.steps[env] + 1.f;
    }
  }
  // The batch-wide broad phase of every substep, inside the kernel.  ARRIVE: the block's pairs-in-range bits go
  // to the global mask of the substep and the block checks in at its barrier, both as reductions that return
  // nothing, so no thread waits on them.  WAIT only where the first masked work item is due — the trigonometry,
  // the per-entity forces and the unmasked items in front of it (sphere pairs) run while the other blocks
  // arrive — and only if the block's own envs left a masked bit unset: the batch-wide mask is the OR of every
  // block's bits, so a block that has them all already holds it.  Substep s uses a.mask + s * (MW + 2): [MW]
  // bits, arrivals; after the epilogue, the last block to finish clears every substep's region for the next step.
  uint32_t mask_words[MW > 0 ? MW : 1];
  [[maybe_unused]] __shared__ uint32_t s_mask[MW > 0 ? MW : 1];   // the block's own bits
  [[maybe_unused]] __shared__ uint32_t s_gmask[MW > 0 ? MW : 1];  // the batch-wide mask, where the block waited
  static_assert(MW <= W::BLOCK, "more mask words than threads in a block");
  uint32_t sig = 0;
  for (int sub = 0; sub < W::cfg.substeps; ++sub) {
    [[maybe_unused]] uint32_t* gmask = a.mask + sub * (MW + 2);
    if constexpr (MW > 0) {
      if (a.use_mask) {
        if (sub > 0) __syncthreads();  // (every thread has taken the previous substep's mask out of s_mask)
        if (threadIdx.x < MW) s_mask[threadIdx.x] = 0u;
        __syncthreads();
        uint32_t bits[MW];
#pragma unroll
        for (int w = 0; w < MW; ++w) bits[w] = 0u;
        // masked items m0, m1 on the even / odd lanes; a warp's even lanes vote for m0, its odd lanes for m1
        static_for<(spec_n_masked<W>() + G - 1) / G>([&](auto ji) {
          constexpr int j0 = decltype(ji)::value * G, j1 = j0 + G - 1 < spec_n_masked<W>() ? j0 + G - 1 : j0;
          constexpr ItemC i0 = W::item[spec_masked_item<W>(j0)], i1 = W::item[spec_masked_item<W>(j1)];
          const bool o = j0 != j1 && odd;
          const bool near = live && norm2((o ? r.px[i1.a] : r.px[i0.a]) - (o ? r.px[i1.b] : r.px[i0.b]),
                                          (o ? r.py[i1.a] : r.py[i0.a]) - (o ? r.py[i1.b] : r.py[i0.b])) <=
                                        (o ? i1.broad_thr : i0.broad_thr);
          if constexpr (j0 == j1) {
            if (__any_sync(0xffffffffu, near)) bits[i0.mask_bit >> 5] |= 1u << (i0.mask_bit & 31);
          } else {
            const unsigned vote = __ballot_sync(0xffffffffu, near);
            if (vote & 0x55555555u) bits[i0.mask_bit >> 5] |= 1u << (i0.mask_bit & 31);
            if (vote & 0xAAAAAAAAu) bits[i1.mask_bit >> 5] |= 1u << (i1.mask_bit & 31);
          }
        });
        if ((threadIdx.x & 31) == 0) {
#pragma unroll
          for (int w = 0; w < MW; ++w)
            if (bits[w]) atomicOr(&s_mask[w], bits[w]);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
          for (int w = 0; w < MW; ++w) {
            const uint32_t b = s_mask[w];
            if (b) red_or_u32(&gmask[w], b);
          }
          red_release_add_u32(&gmask[MW], 1u);
        }
      }
    }
    static_for<(spec_n_trig<W>() + G - 1) / G>([&](auto ki) {
      constexpr int K = decltype(ki)::value;
      float s, c;
      spec_trig_round_eval<W, G, K>(r, odd, s, c);
      if constexpr (G * K + 1 < spec_n_trig<W>() && G > 1)
        spec_trig_round_put<W, G, K>(r, odd, s, c, pair_swap(s), pair_swap(c));
      else
        spec_trig_round_put<W, G, K>(r, odd, s, c, s, c);
    });
    spec_entity_forces<W>(r, afx, afy, atq);
    static_for<R::N>([&](auto ki) {
      constexpr int K = decltype(ki)::value;
      if constexpr (MW > 0 && R::template I0<K> == spec_first_masked<W>()) {
        if (a.use_mask) {  // WAIT
          // (s_mask holds the block's own bits since ARRIVE's __syncthreads and stays put: every thread takes the
          // same branch)
          bool full = true;
          static_for<MW>([&](auto wi) {
            constexpr uint32_t all = spec_mask_full<W>(decltype(wi)::value);
            full = full && s_mask[decltype(wi)::value] == all;
          });
          if (full) {
#pragma unroll
            for (int w = 0; w < MW; ++w) mask_words[w] = s_mask[w];
          } else {
            if (threadIdx.x == 0) {
              while (ld_acquire_u32(&gmask[MW]) < gridDim.x) __nanosleep(20);
              for (int w = 0; w < MW; ++w) s_gmask[w] = s_mask[w] | ld_acquire_u32(&gmask[w]);
            }
            __syncthreads();
#pragma unroll
            for (int w = 0; w < MW; ++w) mask_words[w] = s_gmask[w];
          }
        }
      }
      if constexpr (R::template I0<K> == R::template I1<K>) {  // a lone item: both lanes evaluate it
        spec_item<W, R::template I0<K>, false>(r, a, env, mask_words, sig);
      } else {
        const ItemOut own = spec_round_eval<W, G, K>(r, a, env, mask_words, odd);
        spec_round_add<W, G, K>(r, a, mask_words, own, spec_round_swap<W, G, K>(own), odd);
      }
    });
    spec_integrate<W>(r, sub);
  }
  if (!live) return;
  rows.store(a, env, r, afx, afy, atq, G, odd ? 1 : 0);
  const auto from_lane0 = [odd](float v) {
    if constexpr (G == 1) return v;
    const float v0 = __shfl_xor_sync(0x3u << (threadIdx.x & 30), v, 1);  // (both lanes of a pair are here)
    return odd ? v0 : v;
  };
  if constexpr (epi_counts<P>())
    spec_epilogue<W, P>(r, a, e, env, G, odd ? 1 : 0, from_lane0, [count](const float*) { return count; });
  else
    spec_epilogue<W, P>(r, a, e, env, G, odd ? 1 : 0, from_lane0);
  spec_lidar<W, P, G>(r, a, e, env, odd);
  if constexpr (MW > 0) {
    // thread 0 (always live: it owns the block's first env) is the only thread that touches a.mask.  Once every
    // block has counted itself here, every block has arrived at every barrier and read every mask it waited for,
    // so the last one clears all the regions: the release / acquire of the count orders those reads and
    // arrivals before the clearing stores.
    if (a.use_mask && threadIdx.x == 0) {
      if (atom_acq_rel_add_u32(&a.mask[MW + 1], 1u) == gridDim.x - 1) {
        for (int w = 0; w < W::cfg.substeps * (MW + 2); ++w) a.mask[w] = 0u;
      }
    }
  }
}

// resident blocks of step_env_kernel<W, P, G> on the current device (occupancy query, once per device)
template <class W, class P, int G>
static cudaError_t env_capacity(long& cap) {
  static long capacity[64] = {0};
  int device = 0;
  cudaError_t err = cudaGetDevice(&device);
  if (err != cudaSuccess) return err;
  cap = device < 64 ? capacity[device] : 0;
  if (cap == 0) {
    int per_sm = 0, sms = 0;
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, step_env_kernel<W, P, G>, W::BLOCK * G, 0);
    if (err != cudaSuccess) return err;
    err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err != cudaSuccess) return err;
    cap = (long)per_sm * sms;
    if (device < 64) capacity[device] = cap;
  }
  return cudaSuccess;
}

template <class W, class P, int G>
static cudaError_t launch_env_lanes(const SpecArgs& a, const EpiArgs& e, const ActArgs& act, long blocks, bool coop,
                                    cudaStream_t stream) {
  if (coop) {
    void* args[] = {const_cast<SpecArgs*>(&a), const_cast<EpiArgs*>(&e), const_cast<ActArgs*>(&act)};
    return cudaLaunchCooperativeKernel(reinterpret_cast<void*>(step_env_kernel<W, P, G>), dim3((unsigned)blocks),
                                       dim3(W::BLOCK * G), args, 0, stream);
  }
  step_env_kernel<W, P, G><<<(unsigned)blocks, W::BLOCK * G, 0, stream>>>(a, e, act);
  return cudaGetLastError();
}

// Two lanes per env while every block fits the GPU at once, else one: that holds twice the envs resident, which
// the grid barrier of a masked world needs.  cudaErrorCooperativeLaunchTooLarge: the batch does not fit the GPU
// at once even so (masked worlds only)
template <class W, class P>
static cudaError_t launch_env(const SpecArgs& a, const EpiArgs& e, const ActArgs& act, cudaStream_t stream) {
  for (int k = 0; k < P::N_ACT; ++k)  // (the kernel reads each agent's tensors as what it was compiled for)
    if (act.kind[k] != P::act[k].kind || act.dyn[k] != P::act[k].dyn || act.size[k] != P::act[k].size)
      return cudaErrorInvalidValue;
  if (epi_counts<P>() && !act.steps) return cudaErrorInvalidValue;  // (the program's count comes from the prologue)
  const long blocks = ((long)a.batch_dim + W::BLOCK - 1) / W::BLOCK;
  const bool coop = W::MASK_WORDS > 0 && a.use_mask;
  long cap = 0;
  cudaError_t err = env_capacity<W, P, 2>(cap);
  if (err != cudaSuccess) return err;
  if (blocks <= cap) return launch_env_lanes<W, P, 2>(a, e, act, blocks, coop, stream);
  if (coop) {
    err = env_capacity<W, P, 1>(cap);
    if (err != cudaSuccess) return err;
    if (blocks > cap) return cudaErrorCooperativeLaunchTooLarge;
  }
  return launch_env_lanes<W, P, 1>(a, e, act, blocks, coop, stream);
}

template <class W, class P>
static cudaError_t launch_fused(const SpecArgs& a, const EpiArgs& e, cudaStream_t stream) {
  const long blocks = ((long)a.batch_dim + W::BLOCK - 1) / W::BLOCK;
  step_fused_kernel<W, P><<<(unsigned)blocks, W::BLOCK, 0, stream>>>(a, e);
  return cudaGetLastError();
}

// host-side launcher used by the registry in generated/specializations.cuh
template <class W>
static cudaError_t launch_spec(const SpecArgs& a, cudaStream_t stream) {
  if constexpr (spec_needs_params<W>()) {
    if (!a.ent_params) return cudaErrorInvalidValue;  // (a world with per-env mass / friction needs its table)
  }
  if constexpr (spec_needs_gravity<W>()) {
    if (!a.ent_gravity) return cudaErrorInvalidValue;
  }
  const long blocks = ((long)a.batch_dim + W::BLOCK - 1) / W::BLOCK;
  if (a.order || a.sig)
    step_spec_kernel<W, true><<<(unsigned)blocks, W::BLOCK, 0, stream>>>(a);
  else
    step_spec_kernel<W, false><<<(unsigned)blocks, W::BLOCK, 0, stream>>>(a);
  return cudaGetLastError();
}
#endif  // __CUDACC__

#ifdef __CUDACC__
struct SpecEntry {
  uint64_t hash;
  const char* name;
  int n_entities, n_items;
  cudaError_t (*launch)(const SpecArgs&, cudaStream_t);       // one thread per env (step_spec_kernel)
  cudaError_t (*launch_tile)(const SpecArgs&, cudaStream_t);  // a warp owns a tile of 32 envs, compacted narrow phase
  bool has_tile;                                              // (step_tile_kernel; not for worlds with joints)
};
#endif

}  // namespace vmas
