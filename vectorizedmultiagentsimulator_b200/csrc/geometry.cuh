// geometry.cuh — scalar (one pair, one env) narrow-phase geometry for the VMAS physics kernels.
//
// Each routine is the per-element arithmetic of one batched routine of the reference
// (vmas/simulator/physics.py, cited per function), written for registers:
// segments carry their precomputed unit direction so sin/cos are evaluated once per entity per
// substep.  The file is compiled with -fmad=false: every multiply and add rounds separately,
// like the reference's chain of eager elementwise ops; the only fused operation is inside
// norm2(), which reproduces torch's vector_norm rounding (sqrt(fma(y, y, x*x))).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#ifdef __CUDACC__
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#endif

#define DEVI __device__ __forceinline__

namespace vmas {

// 16-bit observation values (VMAS_DTYPE_F16 / VMAS_DTYPE_BF16): fp32 -> the bits of the 16-bit value, rounded to
// nearest even by the hardware conversion (cvt.rn.f16.f32 / cvt.rn.bf16.f32, packed pairs as cvt.rn.*x2.f32):
// overflow goes to +-inf, -0 stays -0, NaN stays NaN.  x2: `lo` in the low half (the lower address).  The host
// build (tests/hostsim) spells out the same rounding; NaN payloads may differ from the device's.
DEVI uint16_t f16_bits(float v) {
#ifdef __CUDA_ARCH__
  return __half_as_ushort(__float2half_rn(v));
#else
  const uint32_t x = __float_as_uint(v), ax = x & 0x7FFFFFFFu;
  const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
  if (ax > 0x7F800000u) return (uint16_t)(sign | 0x7E00u | ((ax >> 13) & 0x3FFu));
  if (ax >= 0x477FF000u) return (uint16_t)(sign | 0x7C00u);  // >= 65520: the tie above 65504 rounds to inf
  if (ax >= 0x38800000u) {                                  // normal: re-bias the exponent, round 13 bits
    const uint32_t r = ax - 0x38000000u;
    return (uint16_t)(sign | ((r + 0xFFFu + ((r >> 13) & 1u)) >> 13));
  }
  const int e = (int)(ax >> 23);  // subnormal (or zero) in units of 2^-24
  const int shift = 126 - e;
  if (e == 0 || shift > 24) return sign;
  const uint32_t m = (ax & 0x7FFFFFu) | 0x800000u;
  uint32_t q = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1u))) ++q;
  return (uint16_t)(sign | q);
#endif
}
DEVI uint16_t bf16_bits(float v) {
#ifdef __CUDA_ARCH__
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
#else
  const uint32_t x = __float_as_uint(v);
  if ((x & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((x >> 16) | 0x40u);
  return (uint16_t)((x + 0x7FFFu + ((x >> 16) & 1u)) >> 16);
#endif
}
DEVI uint32_t f16x2_bits(float lo, float hi) {
#ifdef __CUDA_ARCH__
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
#else
  return (uint32_t)f16_bits(lo) | ((uint32_t)f16_bits(hi) << 16);
#endif
}
DEVI uint32_t bf16x2_bits(float lo, float hi) {
#ifdef __CUDA_ARCH__
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
#else
  return (uint32_t)bf16_bits(lo) | ((uint32_t)bf16_bits(hi) << 16);
#endif
}
template <int DT>
DEVI uint16_t obs16_bits(float v) {
  static_assert(DT == 1 || DT == 2, "16-bit observation dtypes: VMAS_DTYPE_F16, VMAS_DTYPE_BF16");
  if constexpr (DT == 1) return f16_bits(v);
  else return bf16_bits(v);
}
template <int DT>
DEVI uint32_t obs16x2_bits(float lo, float hi) {
  static_assert(DT == 1 || DT == 2, "16-bit observation dtypes: VMAS_DTYPE_F16, VMAS_DTYPE_BF16");
  if constexpr (DT == 1) return f16x2_bits(lo, hi);
  else return bf16x2_bits(lo, hi);
}

struct V2 {
  float x, y;
};

DEVI V2 mk(float x, float y) { V2 v; v.x = x; v.y = y; return v; }
DEVI V2 operator+(V2 a, V2 b) { return mk(a.x + b.x, a.y + b.y); }
DEVI V2 operator-(V2 a, V2 b) { return mk(a.x - b.x, a.y - b.y); }
DEVI V2 operator*(V2 a, float k) { return mk(a.x * k, a.y * k); }
DEVI V2 neg(V2 a) { return mk(-a.x, -a.y); }

// torch.linalg.vector_norm over a length-2 last dim on CPU rounds as sqrt(fma(y, y, x*x)).
DEVI float norm2(float x, float y) { return sqrtf(__fmaf_rn(y, y, __fmul_rn(x, x))); }
DEVI float norm2(V2 v) { return norm2(v.x, v.y); }
DEVI float dot2(V2 a, V2 b) { return a.x * b.x + a.y * b.y; }           // (a*b).sum(-1)
DEVI float cross2(V2 a, V2 b) { return a.x * b.y - a.y * b.x; }         // ref utils.py:194-197
DEVI float sgnf(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }  // torch.sign
// a / b for a positive divisor.  IEEE division takes a ~100-instruction slow path when the numerator
// is zero (FCHK fails), which is the common case here (contact normals along an axis, resting bodies,
// zero torque) — and a select does not help: the compiler evaluates the division for every lane and
// the lanes with a zero numerator still walk the slow path (measured: 14 % of the balance kernel's
// warp-instructions).  So the division itself is given a harmless numerator (1) in
// that case; (+-0) / b == +-0 for b > 0, so the numerator itself is the exact quotient.
DEVI float div_pos(float a, float b) {
  const bool zero = (a == 0.f && b > 0.f);
  const float q = (zero ? 1.f : a) / b;
  return zero ? a : q;
}
// torch.clamp(x, lo, hi): a NaN stays NaN, where fminf(fmaxf(x, lo), hi) would return a bound and let a
// NaN force, velocity or position carry on as finite state.  Any other x gives fminf(fmaxf(x, lo), hi)'s
// bits, signed zeros included: max.NaN / min.NaN (sm_80+) differ from max / min only in NaN handling.
// The host build (tests/hostsim) spells out the same order, -0 below +0, rather than trust libm's.
DEVI float clampf(float x, float lo, float hi) {
#ifdef __CUDA_ARCH__
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(lo));
  asm("min.NaN.f32 %0, %0, %1;" : "+f"(r) : "f"(hi));
  return r;
#else
  if (x != x) return x;
  const float m = (x > lo || (x == lo && !signbit(x))) ? x : lo;
  return (m < hi || (m == hi && signbit(m))) ? m : hi;
#endif
}
// rotate `v` by the angle whose (cos, sin) is (c, s)  (ref utils.py:176-191)
DEVI V2 rot2(V2 v, float c, float s) { return mk(v.x * c - v.y * s, v.x * s + v.y * c); }

// A segment: centre, unit direction (cos, sin of its angle), half length.
struct Seg {
  V2 p;
  float c, s;
  float half;
};
DEVI Seg mkseg(V2 p, float c, float s, float half) { Seg g; g.p = p; g.c = c; g.s = s; g.half = half; return g; }

// Closest point of a segment to q (ref physics.py:400-429, limit_to_line_length=True).
DEVI V2 closest_point_seg(const Seg& l, V2 q) {
  V2 d = l.p - q;
  float along = d.x * l.c + d.y * l.s;
  // sign(along) * min(|along|, half): multiplying by +-1 is exact, so this is a copysign
  float reach = copysignf(fminf(fabsf(along), l.half), along);
  return mk(l.p.x - reach * l.c, l.p.y - reach * l.s);
}

// Same on the infinite carrier line (limit_to_line_length=False; used by the LIDAR).
DEVI V2 closest_point_carrier(V2 p, float c, float s, V2 q) {
  V2 d = p - q;
  float along = d.x * c + d.y * s;  // sign(along) * |along| == along
  return mk(p.x - along * c, p.y - along * s);
}

struct Pair {
  V2 a, b;
};

// Closest pair of points between two segments (ref physics.py:144-219, 222-260, 132-141).
__device__ __noinline__ Pair closest_seg_seg(const Seg& l1, const Seg& l2) {
  V2 o1 = mk(l1.half * l1.c, l1.half * l1.s);
  V2 o2 = mk(l2.half * l2.c, l2.half * l2.s);
  V2 a1 = l1.p + o1, a2 = l1.p - o1;
  V2 b1 = l2.p + o2, b2 = l2.p - o2;

  // four end-point projections, first strict minimum
  Pair best;
  best.a = mk(INFINITY, INFINITY);
  best.b = mk(INFINITY, INFINITY);
  float dbest = INFINITY;
  {
    V2 q = closest_point_seg(l2, a1);
    float d = norm2(a1 - q);
    if (d < dbest) { dbest = d; best.a = a1; best.b = q; }
  }
  {
    V2 q = closest_point_seg(l2, a2);
    float d = norm2(a2 - q);
    if (d < dbest) { dbest = d; best.a = a2; best.b = q; }
  }
  {
    V2 q = closest_point_seg(l1, b1);
    float d = norm2(q - b1);
    if (d < dbest) { dbest = d; best.a = q; best.b = b1; }
  }
  {
    V2 q = closest_point_seg(l1, b2);
    float d = norm2(q - b2);
    if (d < dbest) { dbest = d; best.a = q; best.b = b2; }
  }
  // proper intersection overrides both points
  V2 r = a2 - a1, s = b2 - b1, qp = b1 - a1;
  float rxs = cross2(r, s);
  float u = cross2(qp, r) / rxs;
  float t = cross2(qp, s) / rxs;
  if (rxs != 0.f && 0.f <= u && u <= 1.f && 0.f <= t && t <= 1.f) {
    V2 x = mk(a1.x + t * r.x, a1.y + t * r.y);
    best.a = x;
    best.b = x;
  }
  return best;
}

// A box in world space: centre, (cos, sin) of its angle and of angle + pi/2, half extents.
struct BoxG {
  V2 p;
  float c, s, c2, s2;
  float half_l, half_w;
};

// Side i of a box as a segment (ref physics.py:298-325): the two `length`-end sides first.
DEVI Seg box_side(const BoxG& b, int i) {
  switch (i) {
    case 0: return mkseg(mk(b.p.x + b.c * b.half_l, b.p.y + b.s * b.half_l), b.c2, b.s2, b.half_w);
    case 1: return mkseg(mk(b.p.x - b.c * b.half_l, b.p.y - b.s * b.half_l), b.c2, b.s2, b.half_w);
    case 2: return mkseg(mk(b.p.x + b.c2 * b.half_w, b.p.y + b.s2 * b.half_w), b.c, b.s, b.half_l);
    default: return mkseg(mk(b.p.x - b.c2 * b.half_w, b.p.y - b.s2 * b.half_w), b.c, b.s, b.half_l);
  }
}

// Closest point on the outline of a box to q (ref physics.py:263-295, 385-397): first strict
// minimum over the four sides.  A side whose distance exceeds the smallest one by a clear margin
// can never be that minimum, so it is skipped on the strength of a cheap box-frame estimate
// (a^2 > 2 a_min^2 + 2 m^2  =>  a > a_min + m); the surviving sides are evaluated exactly and in
// the reference's order, which leaves the result bit-identical.
DEVI V2 closest_point_box(const BoxG& b, V2 q) {
  V2 best = mk(INFINITY, INFINITY);
  float dbest = INFINITY;
  float est[4];
  {
    V2 d = q - b.p;
    float lx = d.x * b.c + d.y * b.s, ly = d.y * b.c - d.x * b.s;
    float ex = fmaxf(fabsf(lx) - b.half_l, 0.f), ey = fmaxf(fabsf(ly) - b.half_w, 0.f);
    float dx0 = lx - b.half_l, dx1 = lx + b.half_l, dy2 = ly - b.half_w, dy3 = ly + b.half_w;
    est[0] = dx0 * dx0 + ey * ey;
    est[1] = dx1 * dx1 + ey * ey;
    est[2] = dy2 * dy2 + ex * ex;
    est[3] = dy3 * dy3 + ex * ex;
  }
  const float keep = 2.f * fminf(fminf(est[0], est[1]), fminf(est[2], est[3])) + 2e-6f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (est[i] > keep) continue;
    Seg sd = box_side(b, i);
    V2 p = closest_point_seg(sd, q);
    float d = norm2(q - p);
    if (d < dbest) { dbest = d; best = p; }
  }
  return best;
}

// Closest (point on box, point on segment) (ref physics.py:328-382): first strict minimum over the
// four sides of the segment/segment result.  Sides are pruned exactly like in closest_point_box:
// in the box frame, lo[i] is a lower bound of the distance between the segment and side i (axis
// separation), up an upper bound of the final minimum (an end point of the segment projected on
// a side is one of the candidates the segment/segment routine considers); a side with
// lo^2 > 2 up^2 + 2 m^2 cannot be the minimum and is skipped.
DEVI Pair closest_box_seg(const BoxG& b, const Seg& l) {
  Pair best;
  best.a = mk(INFINITY, INFINITY);
  best.b = mk(INFINITY, INFINITY);
  float dbest = INFINITY;
  unsigned skip = 0u;  // bit i: side i cannot be the minimum
  {
    V2 d = l.p - b.p;
    const float cx = d.x * b.c + d.y * b.s, cy = d.y * b.c - d.x * b.s;          // segment centre, box frame
    const float ux = l.half * (l.c * b.c + l.s * b.s), uy = l.half * (l.s * b.c - l.c * b.s);
    const float x1 = cx + ux, x2 = cx - ux, y1 = cy + uy, y2 = cy - uy;          // end points, box frame
    const float xmin = fminf(x1, x2), xmax = fmaxf(x1, x2), ymin = fminf(y1, y2), ymax = fmaxf(y1, y2);
    // separation of the segment's bounding box from the box's extent along each axis
    const float sepx = fmaxf(fmaxf(xmin - b.half_l, -b.half_l - xmax), 0.f);
    const float sepy = fmaxf(fmaxf(ymin - b.half_w, -b.half_w - ymax), 0.f);
    // distance of the segment's bounding box from each side's carrier line (0 if it straddles it)
    const float g0 = fmaxf(fmaxf(xmin - b.half_l, b.half_l - xmax), 0.f);
    const float g1 = fmaxf(fmaxf(xmin + b.half_l, -b.half_l - xmax), 0.f);
    const float g2 = fmaxf(fmaxf(ymin - b.half_w, b.half_w - ymax), 0.f);
    const float g3 = fmaxf(fmaxf(ymin + b.half_w, -b.half_w - ymax), 0.f);
    const float lo0 = fmaxf(g0, sepy), lo1 = fmaxf(g1, sepy), lo2 = fmaxf(g2, sepx), lo3 = fmaxf(g3, sepx);
    // upper bound: squared distance of either end point to the nearest side
    float u2 = INFINITY;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const float px = k ? x2 : x1, py = k ? y2 : y1;
      const float ex = fmaxf(fabsf(px) - b.half_l, 0.f), ey = fmaxf(fabsf(py) - b.half_w, 0.f);
      const float a0 = px - b.half_l, a1 = px + b.half_l, a2 = py - b.half_w, a3 = py + b.half_w;
      u2 = fminf(u2, fminf(fminf(a0 * a0 + ey * ey, a1 * a1 + ey * ey), fminf(a2 * a2 + ex * ex, a3 * a3 + ex * ex)));
    }
    const float up = 2.f * u2 + 2e-6f;
    skip = (lo0 * lo0 > up ? 1u : 0u) | (lo1 * lo1 > up ? 2u : 0u) | (lo2 * lo2 > up ? 4u : 0u) |
           (lo3 * lo3 > up ? 8u : 0u);
  }
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    if ((skip >> i) & 1u) continue;
    Seg sd = box_side(b, i);
    Pair c = closest_seg_seg(sd, l);
    float d = norm2(c.a - c.b);
    if (d < dbest) { dbest = d; best = c; }
  }
  return best;
}

// Closest (point on box 1, point on box 2) (ref physics.py:26-129): the four sides of box 1
// against box 2, then the four sides of box 2 against box 1; first strict minimum.
DEVI Pair closest_box_box(const BoxG& b1, const BoxG& b2) {
  Pair best;
  best.a = mk(INFINITY, INFINITY);
  best.b = mk(INFINITY, INFINITY);
  float dbest = INFINITY;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    Seg sd = box_side(b1, i);
    Pair c = closest_box_seg(b2, sd);  // c.a on box 2, c.b on the side of box 1
    float d = norm2(c.b - c.a);
    if (d < dbest) { dbest = d; best.a = c.b; best.b = c.a; }
  }
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    Seg sd = box_side(b2, i);
    Pair c = closest_box_seg(b1, sd);  // c.a on box 1, c.b on the side of box 2
    float d = norm2(c.a - c.b);
    if (d < dbest) { dbest = d; best.a = c.a; best.b = c.b; }
  }
  return best;
}

// Point inside a solid box the contact force is measured from, and its depth
// (ref physics.py:13-23, incl. the 2*surface result when outside == surface).
__device__ __noinline__ V2 inner_point_box(V2 outside, V2 surface, V2 box_pos, float* depth) {
  V2 v = surface - outside;
  V2 u = box_pos - surface;
  float vn = norm2(v);
  float xm = div_pos(v.x * u.x + v.y * u.y, vn);
  V2 x = mk(div_pos(v.x, vn) * xm, div_pos(v.y, vn) * xm);
  if (vn == 0.f) {
    x = surface;
    xm = 0.f;
  }
  *depth = fabsf(xm);
  return surface + x;
}

// Soft-plus penalty force on `a` (b receives the negative) (ref core.py:2805-2839).
// k = contact margin, c = force multiplier.  Returns exactly 0 outside the active range, which is
// also what the reference's masks produce.  The live-contact arithmetic (IEEE divisions, expf,
// log1pf) is kept out of line: it is rare, and one shared copy instead of one per unrolled work
// item keeps the specialised kernels' code small enough for the instruction cache.
__device__ __noinline__ V2 constraint_force_live(float dx, float dy, float d, float dmin, float c, float k,
                                                 float sign) {
  float x = div_pos((dmin - d) * sign, k);
  float pen = (fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)))) * k;  // logaddexp(0, x) * k
  float cc = sign * c;
  float denom = d > 0.f ? d : 1e-8f;
  return mk(div_pos(cc * dx, denom) * pen, div_pos(cc * dy, denom) * pen);
}

// The force from the separation vector delta = pa - pb (what constraint_force() forms first).
DEVI V2 constraint_force_delta(V2 delta, float dmin, float c, float k, bool attractive) {
  // |delta|^2 exactly as norm2() forms it.  sqrt is monotone, so s > dmin^2 (1 + 2e-6) implies
  // sqrtf(s) > dmin: the common "far apart" case is decided without the square root.
  const float s = __fmaf_rn(delta.y, delta.y, __fmul_rn(delta.x, delta.x));
  if (!attractive && s > dmin * dmin * 1.000002f) return mk(0.f, 0.f);
  float d = sqrtf(s);
  if (d < 1e-6f) return mk(0.f, 0.f);
  if (attractive ? (d < dmin) : (d > dmin)) return mk(0.f, 0.f);
  return constraint_force_live(delta.x, delta.y, d, dmin, c, k, attractive ? -1.f : 1.f);
}

DEVI V2 constraint_force(V2 pa, V2 pb, float dmin, float c, float k, bool attractive) {
  return constraint_force_delta(pa - pb, dmin, c, k, attractive);
}

// true iff a repulsive constraint_force_delta(delta, dmin, ...) gets past its first early-out
DEVI bool contact_possible(V2 delta, float dmin) {
  const float s = __fmaf_rn(delta.y, delta.y, __fmul_rn(delta.x, delta.x));
  return !(s > dmin * dmin * 1.000002f);
}

}  // namespace vmas
