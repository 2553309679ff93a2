// spec_tile_kernel.cuh — warp-tile variant of the world-specialised substep kernel: the contact
// forces run COMPACTED.
//
// step_spec_kernel gives one thread one env and walks the env's work items in order.  The cheap
// part of an item (is the pair anywhere near contact?) is uniform, but the expensive part (closest
// points of boxes / segments, the soft-plus contact force with its IEEE divisions, expf, log1pf) is
// needed by a different subset of items in every env: a warp executes it once per item that is near
// in ANY of its 32 envs, with ~8 of 32 lanes active (ncu: 60 % of the balance
// kernel's warp-instructions run at 5-13 lanes).
//
// Here a warp owns a tile of 32 envs.  Per substep:
//   P1  lane = env     positions / rotations (registers), sin / cos, the far test of every item
//                      (unrolled, constexpr parameters, as in step_spec_kernel) -> a bit mask of NEAR
//                      items per lane, OR-reduced over the warp so that items near in no env cost two
//                      instructions from here on.
//                      DIRECT kinds (sphere-sphere, line-sphere): the contact's separation vector is
//                      cheap and computed right here; pairs that get past the force's first early-out
//                      are appended to the CONTACT RING (shared memory: delta, dmin, lever arms, result
//                      row; append = warp ballot + prefix popcount).
//                      GEOMETRY kinds (box-sphere, box-line, line-line, box-box): the near (item, env)
//                      pairs are appended to the queue of the item's kind.
//   P2a lane = entry   the geometry queues are drained 32 entries at a time: closest points of one
//                      (item, env) pair per lane, the env's positions / trig read from shared memory
//                      rows, item parameters from a constant-memory table derived from the constexpr
//                      world; the resulting contacts go to the same ring.
//   P2b lane = contact whenever the ring holds 32 contacts, one FULL round of the soft-plus force runs
//                      (one shared copy of the expensive code, all lanes busy); the round writes
//                      (fx, fy[, ta][, tb]) to the item's result rows, column = env.
//   P3  lane = env     velocities / forces are loaded, per-entity forces, then the items' results are
//                      added IN ITEM ORDER (only items that produced a contact: the others contribute
//                      an exact zero, and the accumulators are never -0, so skipping them changes no
//                      bit), integration, write-back.
// Only __syncwarp() separates the phases: warps are independent.
//
// Same device functions (geometry.cuh), same operand values, same per-entity summation order as
// step_spec_kernel => bit-identical results (CPU: tests/hostsim, GPU: tests/test_cabi_gpu.py).
// Worlds with joints are not tiled (they keep step_spec_kernel).
#pragma once
#include "spec_kernel.cuh"

namespace vmas {

constexpr int TILE_LANES = 32;
#ifndef TILE_MAX_WARPS
#define TILE_MAX_WARPS 4
#endif
// resident warps per SM the register allocator must leave room for (65536 / (32 * TILE_MIN_WARPS)
// registers per thread at most)
#ifndef TILE_MIN_WARPS
#define TILE_MIN_WARPS 16
#endif
constexpr int TILE_N_KINDS = 7;   // VMAS_K_JOINT .. VMAS_K_BB
constexpr int TILE_RING = 64;     // contact ring capacity: < 32 waiting + <= 32 appended at once
constexpr int TILE_RING_ROWS = 8;  // dx, dy, dmin, lever a (2), lever b (2), meta

__host__ __device__ constexpr bool tile_kind_is_direct(int k) { return k == VMAS_K_SS || k == VMAS_K_LS; }
__host__ __device__ constexpr bool tile_kind_is_geom(int k) {
  return k == VMAS_K_LL || k == VMAS_K_BS || k == VMAS_K_BL || k == VMAS_K_BB;
}

// dynamic view of one work item for the geometry stage (constant memory)
struct TileItem {
  int a, b;            // entities
  int trig_a, trig_b;  // first trig row (c, s, c2, s2) of the entity, or -1
  int row;             // first result row: fx, fy, then ta (if has_ta), tb (if has_tb)
  int has_ta, has_tb;
  int solid_a, solid_b;
  float dmin, a_h0, a_h1, b_h0, b_h1;
};

// one contact waiting for its force: f0 = constraint_force_delta(delta, dmin); f = neg ? -f0 : f0;
// result rows: f.x, f.y[, cross2(lever_a, f)][, cross2(lever_b, -f)]
struct TileContact {
  float dx, dy, dmin, lax, lay, lbx, lby;
  uint32_t meta;  // lane | row << 5 | neg << 16 | has_ta << 17 | has_tb << 18
};
__host__ __device__ constexpr uint32_t tile_meta(int lane, int row, bool neg, bool has_ta, bool has_tb) {
  return (uint32_t)lane | ((uint32_t)row << 5) | (neg ? 1u << 16 : 0u) | (has_ta ? 1u << 17 : 0u) | (has_tb ? 1u << 18 : 0u);
}

template <class W>
struct TileLayout {
  static constexpr int E = W::E, NI = W::NI;
  __host__ __device__ static constexpr bool is_trig(int e) { return (W::ent[e].flags & VMAS_F_TRIG) != 0; }
  __host__ __device__ static constexpr int trig_slot(int e) {
    int n = 0;
    for (int k = 0; k < e; ++k)
      if (is_trig(k)) ++n;
    return n;
  }
  __host__ __device__ static constexpr int kind_count(int k) {
    int n = 0;
    for (int i = 0; i < NI; ++i)
      if (W::item[i].kind == k) ++n;
    return n;
  }
  __host__ __device__ static constexpr uint64_t kinds_mask(bool geom) {  // bit I: item I is a geometry / direct item
    uint64_t m = 0;
    for (int i = 0; i < NI && i < 64; ++i)
      if (geom ? tile_kind_is_geom(W::item[i].kind) : tile_kind_is_direct(W::item[i].kind)) m |= 1ull << i;
    return m;
  }
  static constexpr uint64_t GEOM_MASK = kinds_mask(true), DIRECT_MASK = kinds_mask(false);
  static constexpr bool HAS_GEOM = GEOM_MASK != 0;
  // state rows (only worlds with geometry items need them): px, py of every entity, then c, s, c2, s2
  // of every trig entity
  static constexpr int N_TRIG = trig_slot(E);
  static constexpr int ROW_TRIG = 2 * E;
  static constexpr int ROWS_STATE = HAS_GEOM ? 2 * E + 4 * N_TRIG : 0;
  __host__ __device__ static constexpr int trig_row(int e) { return is_trig(e) ? ROW_TRIG + 4 * trig_slot(e) : -1; }
  // torque rows exist only where the item kind can produce a torque: sphere-sphere items produce
  // none, and the sphere side (b) of line-sphere / box-sphere items none either.  spec_item adds a
  // literal +0 there, which changes no bit (the accumulators are never -0: they start at +0).
  __host__ __device__ static constexpr bool has_ta(int i) {
    return (W::ent[W::item[i].a].flags & VMAS_F_ROTATABLE) != 0 && W::item[i].kind != VMAS_K_SS;
  }
  __host__ __device__ static constexpr bool has_tb(int i) {
    const int k = W::item[i].kind;
    return (W::ent[W::item[i].b].flags & VMAS_F_ROTATABLE) != 0 && (k == VMAS_K_LL || k == VMAS_K_BL || k == VMAS_K_BB);
  }
  __host__ __device__ static constexpr int res_width(int i) { return 2 + (has_ta(i) ? 1 : 0) + (has_tb(i) ? 1 : 0); }
  __host__ __device__ static constexpr int res_row(int i) {
    int n = 0;
    for (int k = 0; k < i; ++k) n += res_width(k);
    return n;
  }
  static constexpr int ROW_RES = ROWS_STATE;
  static constexpr int ROWS_RES = res_row(NI);
  static constexpr int ROWS = ROWS_STATE + ROWS_RES;
  // then the contact ring (TILE_RING_ROWS rows of TILE_RING words) and the geometry queues (one per
  // kind, capacity = (items of the kind) * 32 entries of 16 bits)
  static constexpr int OFF_RING = ROWS * TILE_LANES;
  static constexpr int OFF_QUEUE = OFF_RING + TILE_RING_ROWS * TILE_RING;
  __host__ __device__ static constexpr int geom_base(int k) {  // in entries
    int n = 0;
    for (int q = 0; q < k; ++q)
      if (tile_kind_is_geom(q)) n += kind_count(q) * TILE_LANES;
    return n;
  }
  static constexpr int QUEUE_ENTRIES = geom_base(TILE_N_KINDS);
  static constexpr int FLOATS = OFF_QUEUE + (QUEUE_ENTRIES + 1) / 2;  // per warp
  static constexpr size_t BYTES = (size_t)FLOATS * sizeof(float);
  // warps per block: as many as fit in the static shared-memory limit (48 KB)
  static constexpr int WARPS = (4 * BYTES <= 48 * 1024 && TILE_MAX_WARPS >= 4)   ? 4
                               : (2 * BYTES <= 48 * 1024 && TILE_MAX_WARPS >= 2) ? 2
                                                                                 : 1;
  static constexpr int MIN_BLOCKS = (TILE_MIN_WARPS / WARPS) > 0 ? TILE_MIN_WARPS / WARPS : 1;
  static constexpr bool SUPPORTED = W::N_JOINTS == 0 && NI > 0 && NI <= 64 && BYTES <= 48 * 1024 && ROWS < 2048;
};

template <class W>
struct TileTable {
  TileItem it[W::NI > 0 ? W::NI : 1];
};

template <class W>
__host__ __device__ constexpr TileTable<W> make_tile_table() {
  using L = TileLayout<W>;
  TileTable<W> t{};
  for (int i = 0; i < W::NI; ++i) {
    const ItemC it = W::item[i];
    const EntC ea = W::ent[it.a], eb = W::ent[it.b];
    TileItem& d = t.it[i];
    d.a = it.a;
    d.b = it.b;
    d.trig_a = L::trig_row(it.a);
    d.trig_b = L::trig_row(it.b);
    d.row = L::ROW_RES + L::res_row(i);
    d.has_ta = L::has_ta(i) ? 1 : 0;
    d.has_tb = L::has_tb(i) ? 1 : 0;
    d.solid_a = (ea.flags & VMAS_F_HOLLOW) ? 0 : 1;
    d.solid_b = (eb.flags & VMAS_F_HOLLOW) ? 0 : 1;
    d.dmin = it.dmin_base;
    d.a_h0 = ea.d0 / 2.f;
    d.a_h1 = ea.d1 / 2.f;
    d.b_h0 = eb.d0 / 2.f;
    d.b_h1 = eb.d1 / 2.f;
  }
  return t;
}

#ifdef __CUDACC__
template <class W>
__constant__ TileTable<W> c_tile_table = make_tile_table<W>();
#define TILE_TABLE(W) c_tile_table<W>
#else
template <class W>
inline const TileTable<W> h_tile_table = make_tile_table<W>();
#define TILE_TABLE(W) h_tile_table<W>
#endif

template <class W>
struct Tile {
  using L = TileLayout<W>;
  static constexpr int E = W::E, NA = W::A, NI = W::NI;
  using Mask = uint64_t;

  // what one lane (= env) keeps in registers between the phases
  struct Lane {
    SpecRows<W> rows;
    EnvRegs<E> r;
    float afx[NA > 0 ? NA : 1], afy[NA > 0 ? NA : 1], atq[NA > 0 ? NA : 1];
    Mask near;  // items whose far test says "near" (active in the broad-phase mask)
    Mask hits;  // items whose result rows P3 must add: direct items with a contact, near geometry items
  };

  DEVI static uint16_t* queue(float* sm) { return reinterpret_cast<uint16_t*>(sm + L::OFF_QUEUE); }
  DEVI static float* ring(float* sm) { return sm + L::OFF_RING; }

  // ---- far test of item I (the condition under which spec_item evaluates the narrow phase) ----------
  template <int I>
  DEVI static bool near_item(const EnvRegs<E>& r) {
    constexpr ItemC it = W::item[I];
    constexpr int A = it.a, B = it.b;
    constexpr EntC ea = W::ent[A], eb = W::ent[B];
    const V2 pa = mk(r.px[A], r.py[A]), pb = mk(r.px[B], r.py[B]);
    if constexpr (it.kind == VMAS_K_SS) {
      return contact_possible(pa - pb, it.dmin_base);  // the first early-out of the force itself
    } else if constexpr (it.kind == VMAS_K_LS) {
      Seg l = spec_seg<W, A>(r);
      return !spec_far_apart(l.p, pb, l.half + it.dmin_base);
    } else if constexpr (it.kind == VMAS_K_LL) {
      Seg l1 = spec_seg<W, A>(r), l2 = spec_seg<W, B>(r);
      return !spec_far_apart(l1.p, l2.p, l1.half + l2.half + it.dmin_base);
    } else if constexpr (it.kind == VMAS_K_BS) {
      BoxG bx = spec_box<W, A>(r);
      V2 d0 = pb - bx.p;
      float lx = d0.x * bx.c + d0.y * bx.s, ly = d0.y * bx.c - d0.x * bx.s;
      return !(fabsf(lx) > bx.half_l + it.dmin_base + SPEC_FAR_MARGIN ||
               fabsf(ly) > bx.half_w + it.dmin_base + SPEC_FAR_MARGIN);
    } else if constexpr (it.kind == VMAS_K_BL) {
      BoxG bx = spec_box<W, A>(r);
      Seg l = spec_seg<W, B>(r);
      V2 d0 = l.p - bx.p;
      float lx = d0.x * bx.c + d0.y * bx.s, ly = d0.y * bx.c - d0.x * bx.s;
      float ex = l.half * fabsf(l.c * bx.c + l.s * bx.s), ey = l.half * fabsf(l.s * bx.c - l.c * bx.s);
      return !(fabsf(lx) - ex > bx.half_l + it.dmin_base + SPEC_FAR_MARGIN ||
               fabsf(ly) - ey > bx.half_w + it.dmin_base + SPEC_FAR_MARGIN);
    } else if constexpr (it.kind == VMAS_K_BB) {
      return !spec_far_apart(pa, pb, ea.circ_r + eb.circ_r + it.dmin_base);
    } else {
      return false;
    }
  }

  // ---- P1: trig, state rows -> shared memory (worlds with geometry items), near mask of this env ----
  DEVI static void p1(float* sm, const int lane, Lane& ln, const SpecArgs& a, const uint32_t* mask_words) {
    EnvRegs<E>& r = ln.r;
    spec_trig<W>(r);
    if constexpr (L::HAS_GEOM) {
      static_for<E>([&](auto ei) {
        constexpr int e = decltype(ei)::value;
        sm[(2 * e) * TILE_LANES + lane] = r.px[e];
        sm[(2 * e + 1) * TILE_LANES + lane] = r.py[e];
        if constexpr (L::is_trig(e)) {
          constexpr int t = L::trig_row(e);
          sm[(t + 0) * TILE_LANES + lane] = r.c[e];
          sm[(t + 1) * TILE_LANES + lane] = r.s[e];
          if constexpr (W::ent[e].shape == VMAS_SHAPE_BOX) {
            sm[(t + 2) * TILE_LANES + lane] = r.c2[e];
            sm[(t + 3) * TILE_LANES + lane] = r.s2[e];
          }
        }
      });
    }
    Mask near = 0;
    static_for<NI>([&](auto ii) {
      constexpr int I = decltype(ii)::value;
      constexpr ItemC it = W::item[I];
      bool active = true;
      if constexpr (it.mask_bit >= 0) {  // batch-wide broad phase (ref core.py:2797-2801): warp-uniform
        if (a.use_mask && !((mask_words[it.mask_bit >> 5] >> (it.mask_bit & 31)) & 1u)) active = false;
      }
      if (active && near_item<I>(r)) near |= (Mask)1 << I;
    });
    ln.near = near;
    ln.hits = near & L::GEOM_MASK;
  }

  // ---- direct kinds: the contact of a NEAR item I of this env, if the force can be non-zero --------
  template <int I>
  DEVI static bool direct_contact(const int lane, const EnvRegs<E>& r, TileContact& c) {
    constexpr ItemC it = W::item[I];
    constexpr int A = it.a, B = it.b;
    constexpr int R0 = L::ROW_RES + L::res_row(I);
    const V2 pa = mk(r.px[A], r.py[A]), pb = mk(r.px[B], r.py[B]);
    c.dmin = it.dmin_base;
    c.lax = c.lay = c.lbx = c.lby = 0.f;
    if constexpr (it.kind == VMAS_K_SS) {
      const V2 delta = pa - pb;  // f = F(pa - pb)
      c.dx = delta.x;
      c.dy = delta.y;
      c.meta = tile_meta(lane, R0, false, false, false);
      return true;  // near already means contact_possible
    } else {        // VMAS_K_LS: a = line, b = sphere; f = -F(pb - cp), ta = cross2(cp - l.p, f)
      Seg l = spec_seg<W, A>(r);
      const V2 cp = closest_point_seg(l, pb);
      const V2 delta = pb - cp;
      const V2 lever = cp - l.p;
      c.dx = delta.x;
      c.dy = delta.y;
      c.lax = lever.x;
      c.lay = lever.y;
      c.meta = tile_meta(lane, R0, true, L::has_ta(I), false);
      return contact_possible(delta, it.dmin_base);
    }
  }

  DEVI static void ring_put(float* sm, const int slot, const TileContact& c) {
    float* rg = ring(sm);
    const int s = slot & (TILE_RING - 1);
    rg[0 * TILE_RING + s] = c.dx;
    rg[1 * TILE_RING + s] = c.dy;
    rg[2 * TILE_RING + s] = c.dmin;
    rg[3 * TILE_RING + s] = c.lax;
    rg[4 * TILE_RING + s] = c.lay;
    rg[5 * TILE_RING + s] = c.lbx;
    rg[6 * TILE_RING + s] = c.lby;
    rg[7 * TILE_RING + s] = __uint_as_float(c.meta);
  }

  // ---- P2b: the force of the contact in ring slot `slot`, written to its result rows -----------------
  DEVI static void contact_force(float* sm, const int slot) {
    constexpr CfgC cfg = W::cfg;
    const float* rg = ring(sm);
    const int s = slot & (TILE_RING - 1);
    const uint32_t meta = __float_as_uint(rg[7 * TILE_RING + s]);
    const int lane = meta & 31u, row = (meta >> 5) & 2047u;
    const V2 f0 = constraint_force_delta(mk(rg[0 * TILE_RING + s], rg[1 * TILE_RING + s]), rg[2 * TILE_RING + s],
                                         cfg.collision_force, cfg.contact_margin, false);
    const V2 f = (meta >> 16) & 1u ? neg(f0) : f0;
    sm[row * TILE_LANES + lane] = f.x;
    sm[(row + 1) * TILE_LANES + lane] = f.y;
    const int has_ta = (meta >> 17) & 1u, has_tb = (meta >> 18) & 1u;
    if (has_ta) sm[(row + 2) * TILE_LANES + lane] = cross2(mk(rg[3 * TILE_RING + s], rg[4 * TILE_RING + s]), f);
    if (has_tb) sm[(row + 2 + has_ta) * TILE_LANES + lane] = cross2(mk(rg[5 * TILE_RING + s], rg[6 * TILE_RING + s]), neg(f));
  }

  // ---- P2a: closest points of one queue entry (kind K is compile-time, the item is not).  Returns
  // true with the contact to evaluate, or writes the item's zero result itself and returns false. ---
  template <int K>
  DEVI static bool geom_contact(float* sm, const unsigned entry, TileContact& c) {
    const int lane = entry & 31u, i = entry >> 5;
    const TileItem& t = TILE_TABLE(W).it[i];
    auto row = [&](int rw) -> float& { return sm[rw * TILE_LANES + lane]; };
    const V2 pa = mk(row(2 * t.a), row(2 * t.a + 1)), pb = mk(row(2 * t.b), row(2 * t.b + 1));
    auto seg_a = [&]() { return mkseg(pa, row(t.trig_a), row(t.trig_a + 1), t.a_h0); };
    auto seg_b = [&]() { return mkseg(pb, row(t.trig_b), row(t.trig_b + 1), t.b_h0); };
    auto box_of = [&](V2 p, int tr, float h0, float h1) {
      BoxG b;
      b.p = p;
      b.c = row(tr);
      b.s = row(tr + 1);
      b.c2 = row(tr + 2);
      b.s2 = row(tr + 3);
      b.half_l = h0;
      b.half_w = h1;
      return b;
    };
    V2 delta = mk(0.f, 0.f), la = mk(0.f, 0.f), lb = mk(0.f, 0.f);
    float dmin = t.dmin;
    bool negate = false;
    if constexpr (K == VMAS_K_LL) {  // f = F(c.a - c.b)
      Seg l1 = seg_a(), l2 = seg_b();
      Pair cc = closest_seg_seg(l1, l2);
      delta = cc.a - cc.b;
      la = cc.a - l1.p;
      lb = cc.b - l2.p;
    } else if constexpr (K == VMAS_K_BS) {  // a = box, b = sphere: f = -F(pb - inner, dmin + d)
      BoxG bx = box_of(pa, t.trig_a, t.a_h0, t.a_h1);
      V2 cp = closest_point_box(bx, pb);
      V2 inner = cp;
      float d = 0.f;
      if (t.solid_a) inner = inner_point_box(pb, cp, bx.p, &d);
      delta = pb - inner;
      dmin = t.dmin + d;
      la = cp - bx.p;
      negate = true;
    } else if constexpr (K == VMAS_K_BL) {  // a = box, b = line: f = F(inner - c.b, dmin + d)
      BoxG bx = box_of(pa, t.trig_a, t.a_h0, t.a_h1);
      Seg l = seg_b();
      Pair cc = closest_box_seg(bx, l);
      V2 inner = cc.a;
      float d = 0.f;
      if (t.solid_a) inner = inner_point_box(cc.b, cc.a, bx.p, &d);
      delta = inner - cc.b;
      dmin = t.dmin + d;
      la = cc.a - bx.p;
      lb = cc.b - l.p;
    } else if constexpr (K == VMAS_K_BB) {  // f = F(in1 - in2, (d1 + d2) + dmin)
      BoxG b1 = box_of(pa, t.trig_a, t.a_h0, t.a_h1), b2 = box_of(pb, t.trig_b, t.b_h0, t.b_h1);
      Pair cc = closest_box_box(b1, b2);
      V2 in1 = cc.a, in2 = cc.b;
      float d1 = 0.f, d2 = 0.f;
      if (t.solid_a) in1 = inner_point_box(cc.b, cc.a, b1.p, &d1);
      if (t.solid_b) in2 = inner_point_box(cc.a, cc.b, b2.p, &d2);
      delta = in1 - in2;
      dmin = (d1 + d2) + t.dmin;
      la = cc.a - b1.p;
      lb = cc.b - b2.p;
    }
    if (!contact_possible(delta, dmin)) {  // the force is an exact zero: so are its torques (+-0)
      row(t.row) = 0.f;
      row(t.row + 1) = 0.f;
      if (t.has_ta) row(t.row + 2) = 0.f;
      if (t.has_tb) row(t.row + 2 + t.has_ta) = 0.f;
      return false;
    }
    c.dx = delta.x;
    c.dy = delta.y;
    c.dmin = dmin;
    c.lax = la.x;
    c.lay = la.y;
    c.lbx = lb.x;
    c.lby = lb.y;
    c.meta = tile_meta(lane, t.row, negate, t.has_ta != 0, t.has_tb != 0);
    return true;
  }

  // ---- P3: per-entity forces, the items' results in item order, integration --------------------------
  DEVI static void p3(const float* sm, const int lane, Lane& ln, const int sub) {
    EnvRegs<E>& r = ln.r;
    spec_entity_forces<W>(r, ln.afx, ln.afy, ln.atq);
    const Mask hits = ln.hits;
    if (hits != 0) {
      static_for<NI>([&](auto ii) {
        constexpr int I = decltype(ii)::value;
        constexpr ItemC it = W::item[I];
        constexpr int A = it.a, B = it.b;
        constexpr EntC ea = W::ent[A], eb = W::ent[B];
        constexpr int R0 = L::ROW_RES + L::res_row(I);
        if ((hits >> I) & 1u) {
          const float fx = sm[R0 * TILE_LANES + lane], fy = sm[(R0 + 1) * TILE_LANES + lane];
          if constexpr (ea.flags & VMAS_F_MOVABLE) {
            r.Fx[A] = r.Fx[A] + fx;
            r.Fy[A] = r.Fy[A] + fy;
          }
          if constexpr (L::has_ta(I)) r.T[A] = r.T[A] + sm[(R0 + 2) * TILE_LANES + lane];
          if constexpr (eb.flags & VMAS_F_MOVABLE) {
            r.Fx[B] = r.Fx[B] + (-fx);
            r.Fy[B] = r.Fy[B] + (-fy);
          }
          if constexpr (L::has_tb(I)) r.T[B] = r.T[B] + sm[(R0 + 2 + (L::has_ta(I) ? 1 : 0)) * TILE_LANES + lane];
        }
      });
    }
    spec_integrate<W>(r, sub);
  }
};

#ifdef __CUDACC__
// One warp = one tile of 32 envs.  `sm` is the warp's private slice of shared memory.
template <class W>
DEVI void tile_warp_step(float* sm, const SpecArgs& a, const long env, const int lane,
                         const uint32_t (&mask_words)[W::MASK_WORDS > 0 ? W::MASK_WORDS : 1]) {
  using T = Tile<W>;
  using L = TileLayout<W>;
  constexpr unsigned FULL = 0xffffffffu;
  const bool valid = env < a.batch_dim;
  const long env_c = valid ? env : (long)a.batch_dim - 1;  // the tail tile: idle lanes shadow the last env
  typename T::Lane ln;
  ln.rows.load_pos_rot(a, env_c);
  ln.rows.unpack_pos_rot(ln.r);
  uint16_t* q = T::queue(sm);
  const unsigned lt = (1u << lane) - 1u;

  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    T::p1(sm, lane, ln, a, mask_words);
    if (!valid) ln.near = ln.hits = 0;
    // items near in no env of the tile are skipped by everything below (warp-uniform test)
    uint64_t any = (uint64_t)__reduce_or_sync(FULL, (unsigned)ln.near);
    if constexpr (W::NI > 32) any |= (uint64_t)__reduce_or_sync(FULL, (unsigned)(ln.near >> 32)) << 32;

    int head = 0, tail = 0;  // the contact ring: slots [head, tail), warp-uniform
    auto append = [&](bool has, const TileContact& c) {
      const unsigned m = __ballot_sync(FULL, has);
      if (m) {
        if (has) T::ring_put(sm, tail + __popc(m & lt), c);
        tail += __popc(m);
        if (tail - head >= TILE_LANES) {  // a full round of the force: every lane busy
          __syncwarp();
          T::contact_force(sm, head + lane);
          head += TILE_LANES;
          __syncwarp();
        }
      }
    };

    if (any) {
      // ---- direct kinds: contacts straight from the registers ------------------------------------------
      static_for<W::NI>([&](auto ii) {
        constexpr int I = decltype(ii)::value;
        if constexpr (tile_kind_is_direct(W::item[I].kind)) {
          if ((any >> I) & 1u) {
            TileContact c;
            bool has = false;
            if ((ln.near >> I) & 1u) has = T::template direct_contact<I>(lane, ln.r, c);
            if (has) ln.hits |= (uint64_t)1 << I;
            append(has, c);
          }
        }
      });
      // ---- geometry kinds: queue the near (item, env) pairs, item-major within the kind ----------------
      if constexpr (L::HAS_GEOM) {
        if (any & L::GEOM_MASK) {
          int cnt[TILE_N_KINDS];
#pragma unroll
          for (int k = 0; k < TILE_N_KINDS; ++k) cnt[k] = 0;
          static_for<W::NI>([&](auto ii) {
            constexpr int I = decltype(ii)::value;
            constexpr int K = W::item[I].kind;
            if constexpr (tile_kind_is_geom(K)) {
              if ((any >> I) & 1u) {
                const bool near = (ln.near >> I) & 1u;
                const unsigned m = __ballot_sync(FULL, near);
                if (near) q[L::geom_base(K) + cnt[K] + __popc(m & lt)] = (uint16_t)((I << 5) | lane);
                cnt[K] += __popc(m);
              }
            }
          });
          __syncwarp();  // state rows and queues are complete
          static_for<TILE_N_KINDS>([&](auto ki) {
            constexpr int K = decltype(ki)::value;
            if constexpr (tile_kind_is_geom(K) && L::kind_count(K) > 0) {
              for (int base = 0; base < cnt[K]; base += TILE_LANES) {
                TileContact c;
                bool has = false;
                if (base + lane < cnt[K]) has = T::template geom_contact<K>(sm, q[L::geom_base(K) + base + lane], c);
                append(has, c);
              }
            }
          });
        }
      }
      // ---- the last, partial round ------------------------------------------------------------------------
      __syncwarp();
      if (head + lane < tail) T::contact_force(sm, head + lane);
      __syncwarp();
    }
    if (sub == a.first_substep) {
      ln.rows.load_rest(a, env_c);
      ln.rows.unpack_rest(ln.r, ln.afx, ln.afy, ln.atq);
    }
    T::p3(sm, lane, ln, sub);
    __syncwarp();  // the next substep's P1 overwrites the rows this substep's entries read
  }
  if (valid) ln.rows.store(a, env, ln.r, ln.afx, ln.afy, ln.atq);
}

template <class W>
__global__ void __launch_bounds__(TileLayout<W>::WARPS * TILE_LANES, TileLayout<W>::MIN_BLOCKS) step_tile_kernel(const SpecArgs a) {
  using L = TileLayout<W>;
  constexpr int MW = W::MASK_WORDS;
  __shared__ float s_tile[L::WARPS * L::FLOATS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long env = ((long)blockIdx.x * L::WARPS + warp) * TILE_LANES + lane;

  uint32_t mask_words[MW > 0 ? MW : 1];
  if constexpr (MW > 0) {
    __shared__ uint32_t s_mask[MW];
    if (a.use_mask) {
      for (int w = threadIdx.x; w < MW; w += L::WARPS * TILE_LANES) s_mask[w] = a.mask[w];
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
  // whole warps beyond the batch have nothing to do (the last partial warp stays: its idle lanes
  // take part in the ballots)
  if (((long)blockIdx.x * L::WARPS + warp) * TILE_LANES >= a.batch_dim) return;
  tile_warp_step<W>(s_tile + warp * L::FLOATS, a, env, lane, mask_words);
}

template <class W>
static cudaError_t launch_tile(const SpecArgs& a, cudaStream_t stream) {
  using L = TileLayout<W>;
  if constexpr (L::SUPPORTED) {
    constexpr int per_block = L::WARPS * TILE_LANES;
    const long blocks = ((long)a.batch_dim + per_block - 1) / per_block;
    step_tile_kernel<W><<<(unsigned)blocks, per_block, 0, stream>>>(a);
    return cudaGetLastError();
  } else {
    return cudaErrorNotSupported;
  }
}
#endif  // __CUDACC__

}  // namespace vmas
