// vmas_b200.cu — sm_90a kernels + C ABI for the VMAS physics hot path (see include/vmas_b200.h).
//
// Kernels
//   step_kernel<G, EPL>   fused substep(s): per-entity forces -> joint/contact work items ->
//                         ordered accumulation -> semi-implicit Euler -> write-back.
//                         G lanes of a warp own one env (lane = entity); work items are spread
//                         over the same lanes in kind-uniform rounds, results staged in shared
//                         memory and summed per entity in the reference's order (deterministic,
//                         no atomics).  Sphere-only worlds run all substeps in one launch with
//                         the state held in registers.
//   step_tpe_kernel       the same substeps with one thread per env, its state in shared memory.
//   step_block_kernel     the same substeps with one block per env, for worlds of up to 1024 entities.
//   broad_phase_kernel    batch-wide activation mask of line/box pairs (ref core.py:2797-2801).
//   cast_rays_kernel      LIDAR: thread per (env, ray), min over target entities.
//   pair_query_kernel /   World.get_distance / is_overlapping / get_distance_from_point.
//   point_query_kernel
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (no fast-math).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "geometry.cuh"
#include "generic_step.cuh"
#include "query.cuh"
#include "ingest.cuh"
#include "rays.cuh"
#include "generated/specializations.cuh"
#include "vmas_b200.h"

namespace vmas {

static thread_local char g_last_error[512] = "";

static int fail(const char* fmt, const char* detail = "") {
  snprintf(g_last_error, sizeof(g_last_error), fmt, detail);
  return -1;
}

#define CUDA_OK(expr)                                                    \
  do {                                                                   \
    cudaError_t _e = (expr);                                             \
    if (_e != cudaSuccess) return fail("CUDA error: %s", cudaGetErrorString(_e)); \
  } while (0)

// ---------------------------------------------------------------------------------------------
// the fused substep kernel
// ---------------------------------------------------------------------------------------------
template <int G, int EPL>
__global__ void __launch_bounds__(128) step_kernel(const StepArgs a) {
  extern __shared__ float smem[];
  constexpr int ES = G * EPL;
  const int EPB = blockDim.x / G;
  const int E = a.cfg.n_entities, NI = a.cfg.n_items, A = a.cfg.n_agents;
  const int grp = threadIdx.x / G, lane = threadIdx.x % G;
  const long env = (long)blockIdx.x * EPB + grp;
  const bool live = env < a.cfg.batch_dim;

  // shared memory carve-up: 7 entity arrays, 4 result arrays, mask words
  float* base = smem;
  EnvShared<1> sh;
  sh.pitch = 1;
  sh.px = base + (size_t)(0 * EPB + grp) * ES;
  sh.py = base + (size_t)(1 * EPB + grp) * ES;
  sh.rot = base + (size_t)(2 * EPB + grp) * ES;
  sh.c = base + (size_t)(3 * EPB + grp) * ES;
  sh.s = base + (size_t)(4 * EPB + grp) * ES;
  sh.c2 = base + (size_t)(5 * EPB + grp) * ES;
  sh.s2 = base + (size_t)(6 * EPB + grp) * ES;
  float* res = base + (size_t)7 * EPB * ES;
  sh.rfx = res + (size_t)(0 * EPB + grp) * NI;
  sh.rfy = res + (size_t)(1 * EPB + grp) * NI;
  sh.rta = res + (size_t)(2 * EPB + grp) * NI;
  sh.rtb = res + (size_t)(3 * EPB + grp) * NI;
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(res + (size_t)4 * EPB * NI);

  if (a.use_mask) {
    for (int w = threadIdx.x; w < a.mask_words; w += blockDim.x) s_mask[w] = a.mask[w];
    __syncthreads();
    // the last block to have copied the mask clears it for the next broad-phase pass
    if (threadIdx.x == 0) {
      __threadfence();
      unsigned done = atomicAdd(&a.mask[a.mask_words], 1u);
      if (done == gridDim.x - 1) {
        for (int w = 0; w < a.mask_words; ++w) a.mask[w] = 0u;
        a.mask[a.mask_words] = 0u;
      }
    }
  }

  // ---- per-lane entity state -----------------------------------------------------------
  float px[EPL], py[EPL], vx[EPL], vy[EPL], rt[EPL], w[EPL];
  float afx[EPL], afy[EPL], atq[EPL];  // action force / torque (agents)
  int flg[EPL];
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int e = lane + j * G;
    flg[j] = 0;
    px[j] = py[j] = vx[j] = vy[j] = rt[j] = w[j] = afx[j] = afy[j] = atq[j] = 0.f;
    if (live && e < E) {
      const size_t idx = (size_t)env * E + e;
      flg[j] = __ldg(a.tb.ent_i32 + e * 4 + 1) | (1 << 30);  // bit 30: slot in use
      const float2 p = reinterpret_cast<const float2*>(a.st.pos)[idx];
      px[j] = p.x;
      py[j] = p.y;
      rt[j] = a.st.rot[idx];
      if (flg[j] & VMAS_F_MOVABLE) {
        const float2 v = reinterpret_cast<const float2*>(a.st.vel)[idx];
        vx[j] = v.x;
        vy[j] = v.y;
      }
      if (flg[j] & VMAS_F_ROTATABLE) w[j] = a.st.ang_vel[idx];
      if (flg[j] & VMAS_F_AGENT) {
        const int ai = __ldg(a.tb.ent_i32 + e * 4 + 2);
        const size_t aidx = (size_t)env * A + ai;
        if (flg[j] & VMAS_F_MOVABLE) {
          const float2 f = reinterpret_cast<const float2*>(a.st.force)[aidx];
          afx[j] = f.x;
          afy[j] = f.y;
        }
        if (flg[j] & VMAS_F_ROTATABLE) atq[j] = a.st.torque[aidx];
      }
    }
  }

  const float sub_dt = a.cfg.sub_dt;
  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    float Fx[EPL], Fy[EPL], T[EPL];
    // ---- phase A: publish geometry, per-entity forces (ref core.py:1995-2004) -------------
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
      const int e = lane + j * G;
      Fx[j] = Fy[j] = T[j] = 0.f;
      if (!(flg[j] >> 30)) continue;
      const float* ef = a.tb.ent_f32 + (size_t)e * VMAS_EF_COLS;
      sh.px[e] = px[j];
      sh.py[e] = py[j];
      sh.rot[e] = rt[j];
      if (flg[j] & VMAS_F_TRIG) {
        float sn, cs;
        sincosf(rt[j], &sn, &cs);
        sh.c[e] = cs;
        sh.s[e] = sn;
        if (__ldg(a.tb.ent_i32 + e * 4) == VMAS_SHAPE_BOX) {
          sincosf(rt[j] + HALF_PI_F, &sn, &cs);
          sh.c2[e] = cs;
          sh.s2[e] = sn;
        }
      }
      const float mass = ent_param(a, flg[j], VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS);
      if (flg[j] & VMAS_F_AGENT) {  // ref core.py:2018-2041
        if (flg[j] & VMAS_F_MOVABLE) {
          if (flg[j] & VMAS_F_MAX_F) {
            const float mx = __ldg(ef + VMAS_EF_MAX_F);
            const float n = norm2(afx[j], afy[j]);
            if (n > mx) {
              afx[j] = (afx[j] / n) * mx;
              afy[j] = (afy[j] / n) * mx;
            }
          }
          if (flg[j] & VMAS_F_F_RANGE) {
            const float r = __ldg(ef + VMAS_EF_F_RANGE);
            afx[j] = clampf(afx[j], -r, r);
            afy[j] = clampf(afy[j], -r, r);
          }
          Fx[j] = Fx[j] + afx[j];
          Fy[j] = Fy[j] + afy[j];
        }
        if (flg[j] & VMAS_F_ROTATABLE) {
          if (flg[j] & VMAS_F_MAX_T) {
            const float mx = __ldg(ef + VMAS_EF_MAX_T);
            const float n = fabsf(atq[j]);  // vector_norm of one element
            if (n > mx) atq[j] = (atq[j] / n) * mx;
          }
          if (flg[j] & VMAS_F_T_RANGE) {
            const float r = __ldg(ef + VMAS_EF_T_RANGE);
            atq[j] = clampf(atq[j], -r, r);
          }
          T[j] = T[j] + atq[j];
        }
      }
      if (flg[j] & VMAS_F_LIN_FRIC) {  // ref core.py:2054-2088
        const float speed = norm2(vx[j], vy[j]);
        if (speed != 0.f) {
          const float cap = ent_param(a, flg[j], VMAS_F_LIN_FRIC_ENV, env, e, VMAS_EP_LIN_FRIC, ef, VMAS_EF_LIN_FRIC) * mass;
          Fx[j] = Fx[j] + (-(vx[j] / speed)) * fminf(cap, (fabsf(vx[j]) / sub_dt) * mass);
          Fy[j] = Fy[j] + (-(vy[j] / speed)) * fminf(cap, (fabsf(vy[j]) / sub_dt) * mass);
        }
      }
      if (flg[j] & VMAS_F_ANG_FRIC) {  // ref core.py:2089-2102
        const float speed = fabsf(w[j]);  // vector_norm of one element
        if (speed != 0.f) {
          const float inertia = ent_inertia(a, flg[j], mass, ef);
          const float cap = ent_param(a, flg[j], VMAS_F_ANG_FRIC_ENV, env, e, VMAS_EP_ANG_FRIC, ef, VMAS_EF_ANG_FRIC) * inertia;
          T[j] = T[j] + (-(w[j] / speed)) * fminf(cap, (fabsf(w[j]) / sub_dt) * inertia);
        }
      }
      if (flg[j] & VMAS_F_MOVABLE) {  // ref core.py:2043-2052
        if (a.cfg.has_world_gravity) {
          Fx[j] = Fx[j] + mass * a.cfg.gravity_x;
          Fy[j] = Fy[j] + mass * a.cfg.gravity_y;
        }
        if (flg[j] & VMAS_F_GRAVITY) {
          Fx[j] = Fx[j] + mass * __ldg(ef + VMAS_EF_GRAV_X);
          Fy[j] = Fy[j] + mass * __ldg(ef + VMAS_EF_GRAV_Y);
        }
        if (flg[j] & VMAS_F_GRAVITY_ENV) {
          const float2 g = reinterpret_cast<const float2*>(a.tb.ent_gravity)[(size_t)env * E + e];
          Fx[j] = Fx[j] + mass * g.x;
          Fy[j] = Fy[j] + mass * g.y;
        }
      }
    }
    __syncwarp();

    // ---- phase B: joint / contact work items, one per lane per round ------------------------
    for (int r = 0; r < a.tb.n_rounds; ++r) {
      const int item = __ldg(a.tb.sched + r * G + lane);
      if (item < 0 || !live) continue;
      bool active = true;
      if (a.use_mask) {
        const int mbit = (__ldg(a.tb.item_i32 + item * 4 + 3) >> 8) - 1;
        if (mbit >= 0) active = (s_mask[mbit >> 5] >> (mbit & 31)) & 1u;
      }
      float fx = 0.f, fy = 0.f, ta = 0.f, tb = 0.f;
      if (active) eval_item(a, sh, item, env, &fx, &fy, &ta, &tb);
      sh.rfx[item] = fx;
      sh.rfy[item] = fy;
      sh.rta[item] = ta;
      sh.rtb[item] = tb;
    }
    __syncwarp();

    // ---- phase C: ordered accumulation (ref core.py:2191-2199) + integration (:2862-2908) ----
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
      const int e = lane + j * G;
      if (!(flg[j] >> 30)) continue;
      const bool movable = flg[j] & VMAS_F_MOVABLE, rotatable = flg[j] & VMAS_F_ROTATABLE;
      if (!movable && !rotatable) continue;
      const int lo = __ldg(a.tb.inc_off + e), hi = __ldg(a.tb.inc_off + e + 1);
      for (int i = lo; i < hi; ++i) {
        const int v = __ldg(a.tb.inc + i);
        const int item = v >> 1;
        if (v & 1) {
          if (movable) {
            Fx[j] = Fx[j] + (-sh.rfx[item]);
            Fy[j] = Fy[j] + (-sh.rfy[item]);
          }
          if (rotatable) T[j] = T[j] + sh.rtb[item];
        } else {
          if (movable) {
            Fx[j] = Fx[j] + sh.rfx[item];
            Fy[j] = Fy[j] + sh.rfy[item];
          }
          if (rotatable) T[j] = T[j] + sh.rta[item];
        }
      }
      const float* ef = a.tb.ent_f32 + (size_t)e * VMAS_EF_COLS;
      const float drag_mult = __ldg(ef + VMAS_EF_DRAG_MULT);
      if (movable) {
        const float mass = ent_param(a, flg[j], VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS);
        if (sub == 0) {
          vx[j] = vx[j] * drag_mult;
          vy[j] = vy[j] * drag_mult;
        }
        vx[j] = vx[j] + div_pos(Fx[j], mass) * sub_dt;
        vy[j] = vy[j] + div_pos(Fy[j], mass) * sub_dt;
        if (flg[j] & VMAS_F_MAX_SPEED) {
          const float mx = __ldg(ef + VMAS_EF_MAX_SPEED);
          const float n = norm2(vx[j], vy[j]);
          if (n > mx) {
            vx[j] = (vx[j] / n) * mx;
            vy[j] = (vy[j] / n) * mx;
          }
        }
        if (flg[j] & VMAS_F_V_RANGE) {
          const float r = __ldg(ef + VMAS_EF_V_RANGE);
          vx[j] = clampf(vx[j], -r, r);
          vy[j] = clampf(vy[j], -r, r);
        }
        px[j] = px[j] + vx[j] * sub_dt;
        py[j] = py[j] + vy[j] * sub_dt;
        if (a.cfg.has_x_semidim) px[j] = clampf(px[j], -a.cfg.x_semidim, a.cfg.x_semidim);
        if (a.cfg.has_y_semidim) py[j] = clampf(py[j], -a.cfg.y_semidim, a.cfg.y_semidim);
      }
      if (rotatable) {
        const float inertia =
            ent_inertia(a, flg[j], ent_param(a, flg[j], VMAS_F_MASS_ENV, env, e, VMAS_EP_MASS, ef, VMAS_EF_MASS), ef);
        if (sub == 0) w[j] = w[j] * drag_mult;
        w[j] = w[j] + div_pos(T[j], inertia) * sub_dt;
        rt[j] = rt[j] + w[j] * sub_dt;
      }
    }
  }

  // ---- write-back: only what can have changed --------------------------------------------------
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int e = lane + j * G;
    if (!(flg[j] >> 30)) continue;
    const size_t idx = (size_t)env * E + e;
    if (flg[j] & VMAS_F_MOVABLE) {
      reinterpret_cast<float2*>(a.st.pos)[idx] = make_float2(px[j], py[j]);
      reinterpret_cast<float2*>(a.st.vel)[idx] = make_float2(vx[j], vy[j]);
    }
    if (flg[j] & VMAS_F_ROTATABLE) {
      a.st.rot[idx] = rt[j];
      a.st.ang_vel[idx] = w[j];
    }
    if (flg[j] & VMAS_F_AGENT) {
      const int ai = __ldg(a.tb.ent_i32 + e * 4 + 2);
      const size_t aidx = (size_t)env * A + ai;
      if ((flg[j] & VMAS_F_MOVABLE) && (flg[j] & (VMAS_F_MAX_F | VMAS_F_F_RANGE)))
        reinterpret_cast<float2*>(a.st.force)[aidx] = make_float2(afx[j], afy[j]);
      if ((flg[j] & VMAS_F_ROTATABLE) && (flg[j] & (VMAS_F_MAX_T | VMAS_F_T_RANGE)))
        a.st.torque[aidx] = atq[j];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// thread-per-env substep kernel
//
// One thread owns one env and walks its entities and work items serially: every instruction does
// useful work for 32 envs (no idle entity lanes, kind switches are warp-uniform because all envs
// share the item table), forces accumulate straight into the per-entity accumulators in the
// reference's order, and no intra-env synchronisation is needed.  The env's state lives in shared
// memory as [field][entity][thread] so a warp always touches 32 consecutive words.
// ---------------------------------------------------------------------------------------------
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) step_tpe_kernel(const StepArgs a) {
  extern __shared__ float smem[];
  const int E = a.cfg.n_entities, NI = a.cfg.n_items, A = a.cfg.n_agents;
  const int tid = threadIdx.x;
  const long env = (long)blockIdx.x * BLOCK + tid;
  const bool live = env < a.cfg.batch_dim;
  float* col = smem + tid;  // this thread's column: field k of entity e at col[(k * E + e) * BLOCK]
#define TF(k, e) col[((k)*E + (e)) * BLOCK]
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + (size_t)T_NF * E * BLOCK);

  if (a.use_mask) {
    for (int w = tid; w < a.mask_words; w += BLOCK) s_mask[w] = a.mask[w];
    __syncthreads();
    if (tid == 0) {  // the last block to have copied the mask clears it for the next pass
      __threadfence();
      unsigned done = atomicAdd(&a.mask[a.mask_words], 1u);
      if (done == gridDim.x - 1) {
        for (int w = 0; w < a.mask_words; ++w) a.mask[w] = 0u;
        a.mask[a.mask_words] = 0u;
      }
    }
  }
  if (!live) return;

  EnvShared<BLOCK> sh;
  sh.pitch = BLOCK;
  sh.px = &TF(T_PX, 0);
  sh.py = &TF(T_PY, 0);
  sh.rot = &TF(T_ROT, 0);
  sh.c = &TF(T_C, 0);
  sh.s = &TF(T_S, 0);
  sh.c2 = &TF(T_C2, 0);
  sh.s2 = &TF(T_S2, 0);
  sh.rfx = sh.rfy = sh.rta = sh.rtb = nullptr;

  const size_t ebase = (size_t)env * E, abase = (size_t)env * A;
  for (int e = 0; e < E; ++e) entity_load<BLOCK>(a, col, E, e, ebase);

  const float sub_dt = a.cfg.sub_dt;
  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    // ---- phase A: trig cache + per-entity forces --------------------------------------------
    for (int e = 0; e < E; ++e) entity_forces<BLOCK>(a, col, E, e, env, ebase, abase, sub_dt);
    // ---- phase B: joints and contacts in the reference's accumulation order -----------------
    for (int item = 0; item < NI; ++item) item_accumulate(a, sh, col, E, item, env, s_mask);
    // ---- phase C: semi-implicit Euler ---------------------------------------------------------
    for (int e = 0; e < E; ++e) entity_integrate<BLOCK>(a, col, E, e, env, sub, sub_dt);
  }
  for (int e = 0; e < E; ++e) entity_store<BLOCK>(a, col, E, e, ebase);
#undef TF
}

// ---------------------------------------------------------------------------------------------
// block-per-env substep kernel (worlds whose thread-per-env layout does not fit in shared memory)
//
// One block owns one env; thread t owns entities t, t + BLOCK, ...  The env's state lives in shared
// memory as [field][entity] (52 B per entity), the broad-phase mask words behind it.  Phase B walks
// each entity's incidence list: every work item is evaluated twice, once by each endpoint's owner,
// which keeps its own side.  That costs one extra evaluation per item and saves the result staging
// and the atomics; each entity's sums have the operands and the order of step_tpe_kernel's, so the
// two kernels produce the same bits.
// ---------------------------------------------------------------------------------------------
constexpr int STEP_BLOCK_THREADS = 128;

__global__ void __launch_bounds__(STEP_BLOCK_THREADS) step_block_kernel(const StepArgs a) {
  constexpr int BLOCK = STEP_BLOCK_THREADS;
  extern __shared__ float smem[];
  const int E = a.cfg.n_entities, A = a.cfg.n_agents;
  const int tid = threadIdx.x;
  const long env = blockIdx.x;  // grid = batch_dim: every block owns a live env
  float* const col = smem;
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + (size_t)T_NF * E);

  if (a.use_mask) {
    for (int w = tid; w < a.mask_words; w += BLOCK) s_mask[w] = a.mask[w];
    __syncthreads();
    if (tid == 0) {  // the last block to have copied the mask clears it for the next pass
      __threadfence();
      unsigned done = atomicAdd(&a.mask[a.mask_words], 1u);
      if (done == gridDim.x - 1) {
        for (int w = 0; w < a.mask_words; ++w) a.mask[w] = 0u;
        a.mask[a.mask_words] = 0u;
      }
    }
  }

  EnvShared<1> sh;
  sh.pitch = 1;
  sh.px = smem + (size_t)T_PX * E;
  sh.py = smem + (size_t)T_PY * E;
  sh.rot = smem + (size_t)T_ROT * E;
  sh.c = smem + (size_t)T_C * E;
  sh.s = smem + (size_t)T_S * E;
  sh.c2 = smem + (size_t)T_C2 * E;
  sh.s2 = smem + (size_t)T_S2 * E;
  sh.rfx = sh.rfy = sh.rta = sh.rtb = nullptr;

  const size_t ebase = (size_t)env * E, abase = (size_t)env * A;
  for (int e = tid; e < E; e += BLOCK) entity_load<1>(a, col, E, e, ebase);
  __syncthreads();

  const float sub_dt = a.cfg.sub_dt;
  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    for (int e = tid; e < E; e += BLOCK) entity_forces<1>(a, col, E, e, env, ebase, abase, sub_dt);
    __syncthreads();  // every entity's trig cache is published
    for (int e = tid; e < E; e += BLOCK) entity_accumulate(a, sh, col, E, e, env, s_mask);
    __syncthreads();  // nobody reads positions any more
    for (int e = tid; e < E; e += BLOCK) entity_integrate<1>(a, col, E, e, env, sub, sub_dt);
    __syncthreads();  // the next substep reads the new positions
  }
  for (int e = tid; e < E; e += BLOCK) entity_store<1>(a, col, E, e, ebase);
}

// ---------------------------------------------------------------------------------------------
// batch-wide broad phase (ref core.py:2797-2801): bit i <- any_env(|pa - pb| <= Ra + Rb)
// ---------------------------------------------------------------------------------------------
DEVI void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// Block = (32 envs, BROAD_SLICES item slices): lane = env, each warp tests every
// BROAD_SLICES-th masked item for its 32 envs (item parameters are warp-uniform), so the chain
// of dependent loads per thread is short and there are B * BROAD_SLICES / 32 warps to hide it.
constexpr int BROAD_SLICES = 8;

// block (32, BROAD_SLICES); `block` = which 32-env tile this block handles
DEVI void broad_phase_body(const StepArgs& a, const long block) {
  extern __shared__ uint32_t s_bits[];
  const int W = a.mask_words;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  for (int w = tid; w < W; w += 32 * BROAD_SLICES) s_bits[w] = 0u;
  __syncthreads();
  const long env = block * 32 + threadIdx.x;
  const bool live = env < a.cfg.batch_dim;
  const int E = a.cfg.n_entities;
  const float2* pos = reinterpret_cast<const float2*>(a.st.pos) + (size_t)(live ? env : 0) * E;
  for (int j = threadIdx.y; j < a.cfg.n_masked; j += BROAD_SLICES) {
    const int item = __ldg(a.tb.masked_items + j);
    const int4 ii = __ldg(reinterpret_cast<const int4*>(a.tb.item_i32) + item);
    const float thr = __ldg(a.tb.item_f32 + (size_t)item * VMAS_IF_COLS + VMAS_IF_BROAD_THR);
    bool near = false;
    if (live) {
      const float2 pa = pos[ii.y], pb = pos[ii.z];
      near = norm2(pa.x - pb.x, pa.y - pb.y) <= thr;
    }
    if (__any_sync(0xffffffffu, near) && threadIdx.x == 0) atomicOr(&s_bits[j >> 5], 1u << (j & 31));
  }
  __syncthreads();
  for (int w = tid; w < W; w += 32 * BROAD_SLICES) {
    const uint32_t b = s_bits[w];
    if (b) atomicOr(&a.mask[w], b);
  }
}

__global__ void __launch_bounds__(32 * BROAD_SLICES) broad_phase_kernel(const StepArgs a) {
  broad_phase_body(a, blockIdx.x);
}

// ---------------------------------------------------------------------------------------------
// LIDAR (ref core.py:1662-1786 and the three shape kernels 1281-1372, 1414-1490, 1544-1626)
// ---------------------------------------------------------------------------------------------
// (one ray against one target: rays.cuh)
template <class TargetAt>
DEVI float cast_one_ray(const RayArgs& a, float ang, int n_targets, TargetAt target_at, size_t env_base) {
  const float2 op = reinterpret_cast<const float2*>(a.st.pos)[env_base + a.src];
  const V2 o = mk(op.x, op.y);
  float best = a.max_range;
  float ds = 0.f, dc = 0.f;
  bool have_dir = false;
  for (int i = 0; i < n_targets; ++i) {
    const int t = target_at(i);
    if (!ray_target_in_reach(a, o, t, env_base)) continue;
    if (!have_dir) {
      sincosf(ang, &ds, &dc);
      have_dir = true;
    }
    best = tmin(best, ray_vs_entity(a, o, ang, dc, ds, t, env_base));
  }
  return best;
}

__global__ void __launch_bounds__(256) cast_rays_kernel(const RayArgs a) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)a.cfg.batch_dim * a.n_rays;
  if (idx >= total) return;
  const long env = idx / a.n_rays;
  const size_t env_base = (size_t)env * a.cfg.n_entities;
  float ang = a.angles[idx];
  if (a.add_rot_of >= 0) ang = ang + a.st.rot[env_base + a.add_rot_of];
  a.out[idx] = cast_one_ray(a, ang, a.n_targets, [&](int i) { return __ldg(a.targets + i); }, env_base);
}

struct RayBatchArgs {
  RayArgs base;              // cfg / tables / state; per-sensor fields are filled per thread
  const int32_t* src;        // [Q]
  const int32_t* target_off; // [Q + 1]
  const int32_t* all_targets;
  const float* range;        // [Q]
  const int64_t* out_off;    // [Q] element offset of (env 0, ray 0) of each sensor, or null
  int64_t out_env_stride;    // elements between consecutive envs of one sensor
  int32_t n_sensors;
  int32_t flags;
};

// Block = (rays, envs): blockDim.x rays of blockDim.y consecutive envs of sensor blockIdx.y.
// Phase A: one thread per env of the block finds the targets within the sensor's reach (a bit per
// target, up to RAY_MASK_BITS; more targets fall back to testing reach per ray).  Phase B: one
// thread per ray; rays of an env without any target in reach store max_range straight away, the
// others take sin/cos once and test only the flagged targets.  Results equal the per-ray
// formulation bit for bit (the reach test is an exact early-out, see ray_target_in_reach).
constexpr int RAY_MASK_WORDS = 2, RAY_MASK_BITS = 32 * RAY_MASK_WORDS;

// SPHERES: the caller's VMAS_RAYS_SPHERE_TARGETS hint — no box / line code in the kernel.
template <bool SPHERES>
__global__ void __launch_bounds__(256) cast_rays_batched_kernel(const RayBatchArgs a) {
  extern __shared__ uint32_t s_reach[];  // [blockDim.y][RAY_MASK_WORDS]
  const int R = a.base.n_rays;
  const int q = blockIdx.y;
  const long env0 = (long)blockIdx.x * blockDim.y;
  RayArgs s = a.base;  // per-thread copy with this sensor's parameters
  s.src = __ldg(a.src + q);
  s.max_range = __ldg(a.range + q);
  const int lo = __ldg(a.target_off + q), n_targets = __ldg(a.target_off + q + 1) - lo;
  const bool masked = n_targets <= RAY_MASK_BITS;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, n_threads = blockDim.x * blockDim.y;
  // this thread's own inputs are requested before phase A so their latency overlaps it
  const long env = env0 + threadIdx.y;
  const bool live = env < s.cfg.batch_dim;
  const size_t env_base = (size_t)(live ? env : 0) * s.cfg.n_entities;
  const float2 op = reinterpret_cast<const float2*>(s.st.pos)[env_base + s.src];
  const float src_rot = s.st.rot[env_base + s.src];
  const float ang0 = threadIdx.x < R ? __ldg(s.angles + q * R + threadIdx.x) : 0.f;
  if (masked) {
    for (int i = tid; i < blockDim.y * RAY_MASK_WORDS; i += n_threads) s_reach[i] = 0u;
    __syncthreads();
    // phase A: one (env, target) reach test per thread, all loads independent
    for (int i = tid; i < (int)blockDim.y * n_targets; i += n_threads) {
      const int e = i / n_targets, ti = i - e * n_targets;
      if (env0 + e < s.cfg.batch_dim) {
        const size_t eb = (size_t)(env0 + e) * s.cfg.n_entities;
        const float2 sp = reinterpret_cast<const float2*>(s.st.pos)[eb + s.src];
        if (ray_target_in_reach(s, mk(sp.x, sp.y), __ldg(a.all_targets + lo + ti), eb))
          atomicOr(&s_reach[e * RAY_MASK_WORDS + (ti >> 5)], 1u << (ti & 31));
      }
    }
  }
  __syncthreads();
  if (!live) return;
  const int64_t base = (a.out_off ? __ldg(a.out_off + q) : (int64_t)q * s.cfg.batch_dim * R) + env * a.out_env_stride;
  const bool flip = a.flags & VMAS_RAYS_RANGE_MINUS_DISTANCE;
  uint32_t bits[RAY_MASK_WORDS] = {};
  bool any = !masked;
  if (masked) {
#pragma unroll
    for (int w = 0; w < RAY_MASK_WORDS; ++w) {
      bits[w] = s_reach[threadIdx.y * RAY_MASK_WORDS + w];
      any |= bits[w] != 0u;
    }
  }
  for (int ray = threadIdx.x; ray < R; ray += blockDim.x) {
    float d = s.max_range;
    if (any) {
      const float ang = (ray == threadIdx.x ? ang0 : __ldg(s.angles + q * R + ray)) + src_rot;
      if (masked) {
        const V2 o = mk(op.x, op.y);
        float ds, dc;
        sincosf(ang, &ds, &dc);
#pragma unroll
        for (int w = 0; w < RAY_MASK_WORDS; ++w) {
          for (uint32_t rest = bits[w]; rest; rest &= rest - 1) {
            const int t = __ldg(a.all_targets + lo + 32 * w + __ffs(rest) - 1);
            if constexpr (SPHERES) {
              const float2 tp = reinterpret_cast<const float2*>(s.st.pos)[env_base + t];
              const float radius = __ldg(s.tb.ent_f32 + (size_t)t * VMAS_EF_COLS + VMAS_EF_D0);
              d = tmin(d, ray_vs_sphere(o, dc, ds, mk(tp.x, tp.y), radius, s.max_range));
            } else {
              d = tmin(d, ray_vs_entity(s, o, ang, dc, ds, t, env_base));
            }
          }
        }
      } else if constexpr (SPHERES) {  // more targets than mask bits: reach test per ray
        const V2 o = mk(op.x, op.y);
        float ds = 0.f, dc = 0.f;
        bool have_dir = false;
        for (int i = 0; i < n_targets; ++i) {
          const int t = __ldg(a.all_targets + lo + i);
          if (!ray_target_in_reach(s, o, t, env_base)) continue;
          if (!have_dir) {
            sincosf(ang, &ds, &dc);
            have_dir = true;
          }
          const float2 tp = reinterpret_cast<const float2*>(s.st.pos)[env_base + t];
          const float radius = __ldg(s.tb.ent_f32 + (size_t)t * VMAS_EF_COLS + VMAS_EF_D0);
          d = tmin(d, ray_vs_sphere(o, dc, ds, mk(tp.x, tp.y), radius, s.max_range));
        }
      } else {
        d = cast_one_ray(s, ang, n_targets, [&](int i) { return __ldg(a.all_targets + lo + i); }, env_base);
      }
    }
    s.out[base + ray] = flip ? s.max_range - d : d;
  }
}

// ---------------------------------------------------------------------------------------------
// distance / overlap queries (ref core.py:1788-1969)
// ---------------------------------------------------------------------------------------------
struct QueryArgs {
  VmasWorldConfig cfg;
  VmasPlanTables tb;
  VmasState st;
  int32_t a, b, mode;
  const float* point;
  void* out;
};

DEVI EntG load_ent(const QueryArgs& q, int e, size_t env_base) {
  EntG g;
  g.shape = __ldg(q.tb.ent_i32 + e * 4);
  const float2 p = reinterpret_cast<const float2*>(q.st.pos)[env_base + e];
  g.p = mk(p.x, p.y);
  g.rot = q.st.rot[env_base + e];
  g.d0 = __ldg(q.tb.ent_f32 + (size_t)e * VMAS_EF_COLS + VMAS_EF_D0);
  g.d1 = __ldg(q.tb.ent_f32 + (size_t)e * VMAS_EF_COLS + VMAS_EF_D1);
  g.r_plus_lmd = __ldg(q.tb.ent_f32 + (size_t)e * VMAS_EF_COLS + VMAS_EF_R_PLUS_LMD);
  return g;
}

__global__ void __launch_bounds__(256) pair_query_kernel(const QueryArgs q) {
  const long env = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= q.cfg.batch_dim) return;
  const size_t env_base = (size_t)env * q.cfg.n_entities;
  const EntG ga = load_ent(q, q.a, env_base), gb = load_ent(q, q.b, env_base);
  if (q.mode == 0) {
    static_cast<float*>(q.out)[env] = pair_distance(ga, gb);
    return;
  }
  bool over = false;
  const bool box_sphere = (ga.shape == VMAS_SHAPE_BOX && gb.shape == VMAS_SHAPE_SPHERE) ||
                          (gb.shape == VMAS_SHAPE_BOX && ga.shape == VMAS_SHAPE_SPHERE);
  if (overlap_impossible(ga, gb)) {
    over = false;
  } else if (box_sphere) {
    const bool a_is_box = ga.shape == VMAS_SHAPE_BOX;
    over = box_sphere_overlap(a_is_box ? ga : gb, a_is_box ? gb : ga);
  } else {
    over = pair_distance(ga, gb) < 0.f;
  }
  static_cast<uint8_t*>(q.out)[env] = over ? 1 : 0;
}

struct PairBatchArgs {
  QueryArgs base;
  const int32_t* pairs;  // [K, 2]
  int32_t n_pairs;
  int32_t chunk;  // pairs per thread
};

// Thread = env; a block evaluates PAIR_CHUNK pairs for its tile of envs, so the tile's slab rows
// are fetched from L2 once and re-read from L1 for the other pairs (one thread per (pair, env)
// made every pair re-fetch 32 strided sectors per warp).  Stores are coalesced over envs.
constexpr int PAIR_CHUNK = 8;

// Pairs evaluated by one thread: up to PAIR_CHUNK (the tile's slab rows are fetched once and re-read
// from L1), fewer when the batch is small so that at least ~64 Ki threads are in flight.
static int pairs_per_thread(long batch_dim, int n_pairs) {
  const long c = batch_dim * n_pairs / 65536;
  return (int)(c < 1 ? 1 : c > PAIR_CHUNK ? PAIR_CHUNK : c);
}

// Sphere-only pair batches (the caller's VMAS_QUERY_SPHERES hint): a few instructions per pair and a
// tiny code footprint — the general kernel drags the box / line closest-point code along.
__global__ void __launch_bounds__(128) pair_query_spheres_kernel(const PairBatchArgs a) {
  const long env = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long B = a.base.cfg.batch_dim;
  if (env >= B) return;
  const float2* row = reinterpret_cast<const float2*>(a.base.st.pos) + (size_t)env * a.base.cfg.n_entities;
  for (int j = 0; j < a.base.cfg.n_entities; j += 4) prefetch_l1(row + j);
  const int k_end = min(a.n_pairs, (int)(blockIdx.y + 1) * a.chunk);
  for (int k = blockIdx.y * a.chunk; k < k_end; ++k) {
    const long idx = (long)k * B + env;
    const int ia = __ldg(a.pairs + 2 * k), ib = __ldg(a.pairs + 2 * k + 1);
    const float2 pa = row[ia], pb = row[ib];
    const float centre = norm2(pa.x - pb.x, pa.y - pb.y);
    if (a.base.mode == 2) {
      static_cast<float*>(a.base.out)[idx] = centre;
    } else {
      const float ra = __ldg(a.base.tb.ent_f32 + (size_t)ia * VMAS_EF_COLS + VMAS_EF_D0);
      const float rb = __ldg(a.base.tb.ent_f32 + (size_t)ib * VMAS_EF_COLS + VMAS_EF_D0);
      const float d = (centre - ra) - rb;  // ref core.py:1826-1828: (|pa - pb| - ra) - rb
      if (a.base.mode == 0) {
        static_cast<float*>(a.base.out)[idx] = d;
      } else {
        static_cast<uint8_t*>(a.base.out)[idx] = d < 0.f ? 1 : 0;
      }
    }
  }
}

__global__ void __launch_bounds__(128) pair_query_batched_kernel(const PairBatchArgs a) {
  const long env = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long B = a.base.cfg.batch_dim;
  if (env >= B) return;
  const size_t env_base = (size_t)env * a.base.cfg.n_entities;
  // request the env's pos / rot rows up front: the per-pair loads below then hit L1 instead of
  // paying one cold-miss latency per pair, one after the other
  for (int j = 0; j < 2 * a.base.cfg.n_entities; j += 8) prefetch_l1(a.base.st.pos + 2 * env_base + j);
  for (int j = 0; j < a.base.cfg.n_entities; j += 8) prefetch_l1(a.base.st.rot + env_base + j);
  const int k_end = min(a.n_pairs, (int)(blockIdx.y + 1) * a.chunk);
  for (int k = blockIdx.y * a.chunk; k < k_end; ++k) {
    const long idx = (long)k * B + env;
    const int ia = __ldg(a.pairs + 2 * k), ib = __ldg(a.pairs + 2 * k + 1);
    const EntG ga = load_ent(a.base, ia, env_base), gb = load_ent(a.base, ib, env_base);
    if (a.base.mode == 0) {
      static_cast<float*>(a.base.out)[idx] = pair_distance(ga, gb);
    } else if (a.base.mode == 2) {
      static_cast<float*>(a.base.out)[idx] = norm2(ga.p - gb.p);
    } else {
      static_cast<uint8_t*>(a.base.out)[idx] = pair_overlap(ga, gb) ? 1 : 0;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// distance shaping: the reward pattern  dist = |pa - pb|;  rew = prev - dist * factor;  prev <- dist * factor
// (ref scenarios/balance.py:197-214, navigation.py:203-216, transport.py:139-152) for K pairs at once
// ---------------------------------------------------------------------------------------------
struct ShapingArgs {
  const float* pos;
  const int32_t* pairs;  // [K, 2]
  float* prev;           // [K, B] in / out
  float* dist;           // [K, B] or null
  float* rew;            // [K, B]
  float factor;
  int32_t n_pairs, n_entities, batch_dim, chunk;
};

__global__ void __launch_bounds__(128) distance_shaping_kernel(const ShapingArgs a) {
  const long env = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= a.batch_dim) return;
  const float2* row = reinterpret_cast<const float2*>(a.pos) + (size_t)env * a.n_entities;
  for (int j = 0; j < a.n_entities; j += 4) prefetch_l1(row + j);
  const int k_end = min(a.n_pairs, (int)(blockIdx.y + 1) * a.chunk);
  for (int k = blockIdx.y * a.chunk; k < k_end; ++k) {
    const size_t idx = (size_t)k * a.batch_dim + env;
    const float2 pa = row[__ldg(a.pairs + 2 * k)], pb = row[__ldg(a.pairs + 2 * k + 1)];
    const float d = norm2(pa.x - pb.x, pa.y - pb.y);
    const float shaping = d * a.factor;
    if (a.dist) a.dist[idx] = d;
    a.rew[idx] = a.prev[idx] - shaping;
    a.prev[idx] = shaping;
  }
}

__global__ void __launch_bounds__(256) point_query_kernel(const QueryArgs q) {
  const long env = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= q.cfg.batch_dim) return;
  const EntG g = load_ent(q, q.a, (size_t)env * q.cfg.n_entities);
  const float2 pt = reinterpret_cast<const float2*>(q.point)[env];
  static_cast<float*>(q.out)[env] = dist_from_point(g, mk(pt.x, pt.y));
}

// ---------------------------------------------------------------------------------------------
// observation assembly: every slab-derived column of every agent's observation in one launch
// (the reference concatenates per-agent slices with torch.cat, e.g. scenarios/balance.py:236-262)
// ---------------------------------------------------------------------------------------------
struct ObsArgs {
  VmasState st;
  const int32_t* cols;  // [rows * width * 4]
  void* out;            // [rows, B, width] of the launch's DT (fp32, or fp16 / bf16 rounded to nearest even)
  int32_t rows, width, batch_dim, n_entities;
  const float* buffers[VMAS_OBS_MAX_BUFFERS];  // VMAS_OBS_BUFFER columns: fp32 [B] each
};

// A source decoded once per thread: where the field's tile starts in shared memory, the element
// offset inside an env's row, and the row pitch.
struct ObsSrc {
  unsigned base, pitch;
};


// blockIdx.y = observation row, blockIdx.x = a tile of `tile_envs` consecutive envs.
// (1) The tile's slab rows (pos, vel, rot, ang_vel: four contiguous global ranges) are copied to
//     shared memory with coalesced vector loads — reading the scattered columns straight from
//     global memory costs a 32-byte sector per 4-byte value.
// (2) threadIdx.x = a group of VEC adjacent columns, threadIdx.y = env lane: a thread decodes its
//     columns once (shared-memory offsets in registers) and walks the tile's envs; per env a
//     handful of shared-memory loads, at most one subtraction per column and one vector store;
//     consecutive lanes write consecutive pieces of an env's output row.  DT != VMAS_DTYPE_F32: the values are
//     rounded to 16 bits in registers and stored at half the width (4 columns: one 8-byte store).
template <int VEC, int DT = VMAS_DTYPE_F32>
DEVI void gather_observations_body(const ObsArgs& a, const int tile_envs, const int obs_row) {
  extern __shared__ float4 s_state4[];
  float* s_state = reinterpret_cast<float*>(s_state4);
  const unsigned E = (unsigned)a.n_entities;
  const long env0 = (long)blockIdx.x * tile_envs;
  const unsigned n_env = (unsigned)min((long)tile_envs, (long)a.batch_dim - env0);
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, n_threads = blockDim.x * blockDim.y;
  // field f occupies s_state[base_f, base_f + tile_envs * pitch_f); bases are multiples of 4 floats
  // (scalars, not arrays: dynamically indexed arrays would live in local memory)
  const unsigned T = (unsigned)tile_envs;
  const unsigned base_vel = (T * 2 * E + 3u) & ~3u;
  const unsigned base_rot = base_vel + ((T * 2 * E + 3u) & ~3u);
  const unsigned base_w = base_rot + ((T * E + 3u) & ~3u);
  auto stage = [&](const float* field, unsigned pitch, unsigned base) {
    const float* src = field + (size_t)env0 * pitch;  // 16-byte aligned: env0 * pitch is a multiple of 4
    const unsigned n = n_env * pitch;
    for (unsigned i = 4 * tid; i < n; i += 4 * n_threads) {
      if (i + 4 <= n) {
        *reinterpret_cast<float4*>(s_state + base + i) = *reinterpret_cast<const float4*>(src + i);
      } else {
        for (unsigned k = i; k < n; ++k) s_state[base + k] = src[k];
      }
    }
  };
  stage(a.st.pos, 2 * E, 0u);
  stage(a.st.vel, 2 * E, base_vel);
  stage(a.st.rot, E, base_rot);
  stage(a.st.ang_vel, E, base_w);
  auto decode = [&](int code) {
    const int field = (code >> 24) & 3;
    const unsigned off = (unsigned)(code & 0xFFFFFF);
    ObsSrc r;
    r.base = off + (field == VMAS_OBS_POS ? 0u : field == VMAS_OBS_VEL ? base_vel : field == VMAS_OBS_ROT ? base_rot : base_w);
    r.pitch = field <= VMAS_OBS_VEL ? 2 * E : E;
    return r;
  };
  __syncthreads();

  const int groups = a.width / VEC;
  const int g = threadIdx.x;
  const int row = obs_row;
  const int4* table = reinterpret_cast<const int4*>(a.cols) + (size_t)row * a.width + g * VEC;
  int op[VEC];
  ObsSrc sa[VEC], sb[VEC];
  float par[VEC];
  bool any = false, all = true;
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const int4 c = __ldg(table + k);
    op[k] = c.x;
    sa[k] = decode(c.y);
    sb[k] = decode(c.z);
    if (c.x == VMAS_OBS_BUFFER) sa[k].pitch = (unsigned)c.y & (VMAS_OBS_MAX_BUFFERS - 1);  // (which buffer)
    par[k] = __int_as_float(c.w);
    any |= c.x != VMAS_OBS_SKIP;
    all &= c.x != VMAS_OBS_SKIP;
  }
  if (g >= groups || !any) return;  // columns owned by another producer (LIDAR, the scenario)
  const size_t out_at = ((size_t)row * a.batch_dim + env0) * a.width + g * VEC;
  for (unsigned e = threadIdx.y; e < n_env; e += blockDim.y) {
    float v[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      v[k] = 0.f;
      if (op[k] == VMAS_OBS_BUFFER) {
        v[k] = a.buffers[sa[k].pitch][env0 + e];
      } else if (op[k] != VMAS_OBS_SKIP) {
        v[k] = s_state[sa[k].base + e * sa[k].pitch];
        if (op[k] == VMAS_OBS_DIFF) v[k] = v[k] - s_state[sb[k].base + e * sb[k].pitch];
        if (op[k] == VMAS_OBS_REMAINDER) v[k] = obs_remainder(v[k], par[k]);
      }
    }
    if constexpr (DT == VMAS_DTYPE_F32) {
      float* dst = static_cast<float*>(a.out) + out_at + (size_t)e * a.width;
      if (all) {
        if constexpr (VEC == 4) {
          *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else if constexpr (VEC == 2) {
          *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
        } else {
          dst[0] = v[0];
        }
      } else {
#pragma unroll
        for (int k = 0; k < VEC; ++k)
          if (op[k] != VMAS_OBS_SKIP) dst[k] = v[k];
      }
    } else {
      uint16_t* dst = static_cast<uint16_t*>(a.out) + out_at + (size_t)e * a.width;
      if (all && VEC > 1) {
        if constexpr (VEC == 4) {
          *reinterpret_cast<uint2*>(dst) = make_uint2(obs16x2_bits<DT>(v[0], v[1]), obs16x2_bits<DT>(v[2], v[3]));
        } else if constexpr (VEC == 2) {
          *reinterpret_cast<uint32_t*>(dst) = obs16x2_bits<DT>(v[0], v[1]);
        }
      } else {
#pragma unroll
        for (int k = 0; k < VEC; ++k)
          if (op[k] != VMAS_OBS_SKIP) dst[k] = obs16_bits<DT>(v[k]);
      }
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(256) gather_observations_kernel(const ObsArgs a, const int tile_envs) {
  gather_observations_body<VEC>(a, tile_envs, blockIdx.y);
}

// The observation launches stage a tile of envs' slab rows in shared memory: a multiple of 4 envs (keeps every
// field's tile 16-byte aligned) whose state fits 32 KB.  Past ~500 entities even 4 envs need more than the
// default 48 KB; the launch then opts into more dynamic shared memory, up to VMAS_BLOCK_MAX_ENTITIES.
static int obs_tile(int n_entities, int* tile_out, size_t* smem_out) {
  if (n_entities > VMAS_BLOCK_MAX_ENTITIES) return fail("observation rows of worlds with more than 1024 entities%s");
  const size_t per_env = 6u * (size_t)n_entities * sizeof(float);
  int tile = 128;
  while (tile > 4 && tile * per_env + 64 > 32 * 1024) tile /= 2;
  *tile_out = tile;
  *smem_out = tile * per_env + 64;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// post-step program: the scenario's reward / done glue as ONE launch together with the observation
// gather.  A scenario's callbacks are a handful of distance / overlap queries, the distance-shaping
// pattern and a few elementwise operations on [B] tensors (ref scenarios/balance.py:197-263,
// transport.py:139-190): in torch every one of them is a kernel launch of a few microseconds.  Here they
// are a short instruction list interpreted by one thread per env (registers = per-env scalars, bools as
// 0 / 1), in the blocks with blockIdx.y == obs.rows of a launch whose other blocks assemble the
// observations (horizontal fusion: the two jobs do not depend on each other).
// ---------------------------------------------------------------------------------------------
struct ProgArgs {
  QueryArgs base;  // cfg, plan tables, state
  VmasStepProgram prog;
};

DEVI void post_step_program_body(const ProgArgs& p, const int tile_envs) {
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, n_threads = blockDim.x * blockDim.y;
  const long B = p.base.cfg.batch_dim;
  const long env_end = min(B, ((long)blockIdx.x + 1) * tile_envs);
  for (long env = (long)blockIdx.x * tile_envs + tid; env < env_end; env += n_threads) {
    const size_t env_base = (size_t)env * p.base.cfg.n_entities;
    const float2* row = reinterpret_cast<const float2*>(p.base.st.pos) + env_base;
    // request the env's pos / rot rows up front: the queries below then hit L1 instead of paying one
    // cold-miss latency each, one after the other
    for (int j = 0; j < 2 * p.base.cfg.n_entities; j += 8) prefetch_l1(p.base.st.pos + 2 * env_base + j);
    for (int j = 0; j < p.base.cfg.n_entities; j += 8) prefetch_l1(p.base.st.rot + env_base + j);
    float r[VMAS_PROG_REGS];
#pragma unroll
    for (int i = 0; i < VMAS_PROG_REGS; ++i) r[i] = 0.f;
    for (int pc = 0; pc < p.prog.n_instr; ++pc) {
      const VmasProgInstr in = p.prog.instr[pc];
      const int ia = in.arg & 0xFFFF, ib = (in.arg >> 16) & 0xFFFF;
      switch (in.op) {
        case VMAS_OP_OVERLAP: {
          const EntG ga = load_ent(p.base, ia, env_base), gb = load_ent(p.base, ib, env_base);
          r[in.dst] = pair_overlap(ga, gb) ? 1.f : 0.f;
        } break;
        case VMAS_OP_DISTANCE: {
          const EntG ga = load_ent(p.base, ia, env_base), gb = load_ent(p.base, ib, env_base);
          r[in.dst] = pair_distance(ga, gb);
        } break;
        case VMAS_OP_CENTER_DISTANCE: {
          const float2 pa = row[ia], pb = row[ib];
          r[in.dst] = norm2(pa.x - pb.x, pa.y - pb.y);
        } break;
        case VMAS_OP_SHAPING: {  // dist -> r[dst + 1]; rew = prev - dist * factor -> r[dst]; prev <- dist * factor
          const float2 pa = row[ia], pb = row[ib];
          const float d = norm2(pa.x - pb.x, pa.y - pb.y);
          const float shaping = d * in.imm;
          float* prev = static_cast<float*>(p.prog.buffers[in.a]) + env;
          r[in.dst] = *prev - shaping;
          r[in.dst + 1] = d;
          *prev = shaping;
        } break;
        case VMAS_OP_LOAD_F32:
        case VMAS_OP_STEP_COUNT:  // (the ingest launch in front of this one has counted the step)
          r[in.dst] = static_cast<const float*>(p.prog.buffers[in.a])[env];
          break;
        case VMAS_OP_LOAD_BOOL: r[in.dst] = static_cast<const uint8_t*>(p.prog.buffers[in.a])[env] ? 1.f : 0.f; break;
        case VMAS_OP_CONST: r[in.dst] = in.imm; break;
        case VMAS_OP_ADD: r[in.dst] = r[in.a] + r[in.b]; break;
        case VMAS_OP_SUB: r[in.dst] = r[in.a] - r[in.b]; break;
        case VMAS_OP_MUL: r[in.dst] = r[in.a] * r[in.b]; break;
        case VMAS_OP_MIN: r[in.dst] = fminf(r[in.a], r[in.b]); break;
        case VMAS_OP_MAX: r[in.dst] = fmaxf(r[in.a], r[in.b]); break;
        case VMAS_OP_NEG: r[in.dst] = -r[in.a]; break;
        case VMAS_OP_OR: r[in.dst] = (r[in.a] != 0.f || r[in.b] != 0.f) ? 1.f : 0.f; break;
        case VMAS_OP_AND: r[in.dst] = (r[in.a] != 0.f && r[in.b] != 0.f) ? 1.f : 0.f; break;
        case VMAS_OP_NOT: r[in.dst] = r[in.a] != 0.f ? 0.f : 1.f; break;
        case VMAS_OP_LT: r[in.dst] = r[in.a] < r[in.b] ? 1.f : 0.f; break;
        case VMAS_OP_LE: r[in.dst] = r[in.a] <= r[in.b] ? 1.f : 0.f; break;
        case VMAS_OP_WHERE: r[in.dst] = r[in.a] != 0.f ? r[in.b] : r[in.arg & 0xFF]; break;
        case VMAS_OP_STORE_F32: static_cast<float*>(p.prog.buffers[in.b])[env] = r[in.a]; break;
        case VMAS_OP_STORE_BOOL: static_cast<uint8_t*>(p.prog.buffers[in.b])[env] = r[in.a] != 0.f ? 1 : 0; break;
        default: break;
      }
    }
  }
}

// blockIdx.y == 0 (when there is a program): the program blocks — scheduled first, because a program thread
// is a chain of dependent queries (latency) that the bandwidth-bound gather blocks behind it can hide
template <int VEC, int DT = VMAS_DTYPE_F32>
__global__ void __launch_bounds__(256, 5) post_step_kernel(const ObsArgs obs, const int tile_envs, const ProgArgs prog) {
  const int first_obs = prog.prog.n_instr > 0 ? 1 : 0;
  if ((int)blockIdx.y < first_obs)
    post_step_program_body(prog, tile_envs);
  else
    gather_observations_body<VEC, DT>(obs, tile_envs, (int)blockIdx.y - first_obs);
}

template <bool KIN>
__global__ void __launch_bounds__(256) ingest_actions_kernel(const IngestArgs a) {
  ingest_actions_body<KIN>(a, (long)blockIdx.x * blockDim.x + threadIdx.x);
}

// Action ingest and the first substep's broad phase in ONE launch (blocks [0, n_ingest) ingest, the rest
// test the masked pairs): both only read what the previous step left, neither depends on the other, and
// each is too small to fill the GPU on its own.  Block = (32, BROAD_SLICES) = 256 threads.
static_assert(32 * BROAD_SLICES == 256, "the fused launch assumes 256-thread blocks");
template <bool KIN>
__global__ void __launch_bounds__(256) ingest_broad_kernel(const IngestArgs ia, const StepArgs sa, const int n_ingest) {
  if ((int)blockIdx.x < n_ingest)
    ingest_actions_body<KIN>(ia, (long)blockIdx.x * 256 + threadIdx.y * 32 + threadIdx.x);
  else
    broad_phase_body(sa, (long)blockIdx.x - n_ingest);
}

// PID velocity controller (ref controllers/velocity_controller.py:88-125): one thread per (env, axis)
struct PidArgs {
  const float* vel;
  float *u, *accum, *prev;
  int entity, n_entities, batch_dim;
  float gain, inv_ti, td, dt, windup, mass;
};
__global__ void __launch_bounds__(256) velocity_controller_kernel(const PidArgs a) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)a.batch_dim * 2) return;
  const long env = idx >> 1;
  const int axis = (int)(idx & 1);
  const float err = a.u[idx] - a.vel[((size_t)env * a.n_entities + a.entity) * 2 + axis];
  float sum = err;
  if (a.inv_ti != 0.f) {
    float acc = a.accum[idx] + a.dt * err;
    if (a.windup >= 0.f) acc = fminf(fmaxf(acc, -a.windup), a.windup);
    a.accum[idx] = acc;
    sum = sum + a.inv_ti * acc;
  }
  const float rate = a.td * (err - a.prev[idx]) / a.dt;
  a.prev[idx] = err;
  a.u[idx] = (a.gain * (sum + rate)) * a.mass;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int check_common(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st) {
  if (!cfg || !tb || !st) return fail("null argument%s");
  if (cfg->batch_dim <= 0 || cfg->n_entities <= 0) return fail("empty world%s");
  if (!st->pos || !st->vel || !st->rot || !st->ang_vel) return fail("null state pointer%s");
  if (!tb->ent_f32 || !tb->ent_i32) return fail("null entity tables%s");
  return 0;
}

template <int G, int EPL>
static int launch_step(const StepArgs& args, cudaStream_t stream) {
  const int E = args.cfg.n_entities, NI = args.cfg.n_items;
  if (E > G * EPL) return fail("internal: entity count exceeds the lane layout%s");
  // shrink the block (fewer envs per block) until the result staging fits in shared memory
  int device = 0;
  CUDA_OK(cudaGetDevice(&device));
  static int max_optin[64] = {0};
  if (device < 64 && max_optin[device] == 0)
    CUDA_OK(cudaDeviceGetAttribute(&max_optin[device], cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t limit = device < 64 ? (size_t)max_optin[device] : 48 * 1024;
  int threads = 128;
  size_t smem = 0;
  for (;;) {
    const int epb = threads / G;
    smem = ((size_t)7 * epb * G * EPL + (size_t)4 * epb * NI) * sizeof(float) +
           (size_t)(args.use_mask ? args.mask_words : 0) * sizeof(uint32_t);
    if (smem <= limit || threads <= G) break;
    threads /= 2;
  }
  if (smem > limit) return fail("world too large: work items do not fit in shared memory%s");
  static size_t configured[64] = {0};
  auto kern = step_kernel<G, EPL>;
  if (smem > 48 * 1024 && (device >= 64 || configured[device] < smem)) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
    if (device < 64) configured[device] = limit;
  }
  const int epb = threads / G;
  const long blocks = ((long)args.cfg.batch_dim + epb - 1) / epb;
  kern<<<(unsigned)blocks, threads, smem, stream>>>(args);
  CUDA_OK(cudaGetLastError());
  return 1;
}

template <int BLOCK>
static int launch_tpe(const StepArgs& args, cudaStream_t stream, size_t limit, int device) {
  const size_t smem = (size_t)T_NF * args.cfg.n_entities * BLOCK * sizeof(float) +
                      (size_t)(args.use_mask ? args.mask_words : 0) * sizeof(uint32_t);
  if (smem > limit) return -2;  // caller tries a smaller block
  auto kern = step_tpe_kernel<BLOCK>;
  static size_t configured[64] = {0};
  if (smem > 48 * 1024 && (device >= 64 || configured[device] < smem)) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
    if (device < 64) configured[device] = limit;
  }
  const long blocks = ((long)args.cfg.batch_dim + BLOCK - 1) / BLOCK;
  kern<<<(unsigned)blocks, BLOCK, smem, stream>>>(args);
  CUDA_OK(cudaGetLastError());
  return 1;
}

static int dispatch_tpe(const StepArgs& args, cudaStream_t stream) {
  int device = 0;
  CUDA_OK(cudaGetDevice(&device));
  static int max_optin[64] = {0};
  if (device < 64 && max_optin[device] == 0)
    CUDA_OK(cudaDeviceGetAttribute(&max_optin[device], cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t limit = device < 64 ? (size_t)max_optin[device] : 48 * 1024;
  int r = launch_tpe<64>(args, stream, limit, device);
  if (r == -2) r = launch_tpe<32>(args, stream, limit, device);
  if (r == -2) return fail("world too large: an env's state does not fit in shared memory%s");
  return r;
}

static int launch_block(const StepArgs& args, cudaStream_t stream) {
  if (args.cfg.n_entities > VMAS_BLOCK_MAX_ENTITIES)
    return fail("world too large: the block-per-env step takes at most 1024 entities%s");
  int device = 0;
  CUDA_OK(cudaGetDevice(&device));
  static int max_optin[64] = {0};
  if (device < 64 && max_optin[device] == 0)
    CUDA_OK(cudaDeviceGetAttribute(&max_optin[device], cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t limit = device < 64 ? (size_t)max_optin[device] : 48 * 1024;
  const size_t smem = (size_t)T_NF * args.cfg.n_entities * sizeof(float) +
                      (size_t)(args.use_mask ? args.mask_words : 0) * sizeof(uint32_t);
  if (smem > limit) return fail("world too large: an env's state does not fit in shared memory%s");
  static size_t configured[64] = {0};
  if (smem > 48 * 1024 && (device >= 64 || configured[device] < smem)) {
    CUDA_OK(cudaFuncSetAttribute(step_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
    if (device < 64) configured[device] = limit;
  }
  step_block_kernel<<<(unsigned)args.cfg.batch_dim, STEP_BLOCK_THREADS, smem, stream>>>(args);
  CUDA_OK(cudaGetLastError());
  return 1;
}

// specialisations compiled at run time (vmas_b200_register_specialization): indices kNumSpecs, ...
static SpecEntry g_dyn_specs[VMAS_MAX_RUNTIME_SPECS];
static int g_num_dyn_specs = 0;
static int num_specs() { return kNumSpecs + g_num_dyn_specs; }
static const SpecEntry& spec_at(int index) { return index < kNumSpecs ? kSpecs[index] : g_dyn_specs[index - kNumSpecs]; }

// whole-step kernels compiled at run time (vmas_b200_register_step_kernel): handles 1, 2, ...
struct FusedEntry {
  uint64_t key;
  int n_entities, n_items;
  cudaError_t (*launch)(const SpecArgs&, const EpiArgs&, cudaStream_t);
  cudaError_t (*launch_env)(const SpecArgs&, const EpiArgs&, const ActArgs&, cudaStream_t);  // or null
};
static FusedEntry g_fused[VMAS_MAX_RUNTIME_SPECS];
static int g_num_fused = 0;

static SpecArgs spec_args_of(const StepArgs& args) {
  SpecArgs sa;
  sa.st = args.st;
  sa.joint_rot = args.tb.joint_rot;
  sa.mask = args.mask;
  sa.batch_dim = args.cfg.batch_dim;
  sa.use_mask = args.use_mask;
  sa.first_substep = args.first_substep;
  sa.n_substeps = args.n_substeps;
  sa.order = nullptr;
  sa.sig = nullptr;
  sa.ent_params = args.ent_params;
  sa.ent_gravity = args.tb.ent_gravity;
  return sa;
}

static int dispatch_fused(const StepArgs& args, int handle, const EpiArgs& epi, cudaStream_t stream) {
  if (handle < 1 || handle > g_num_fused) return fail("unknown whole-step kernel%s");
  const FusedEntry& f = g_fused[handle - 1];
  if (f.n_entities != args.cfg.n_entities || f.n_items != args.cfg.n_items)
    return fail("whole-step kernel does not match the world (stale handle?)%s");
  CUDA_OK(f.launch(spec_args_of(args), epi, stream));
  return 1;
}

static int dispatch_spec(const StepArgs& args, cudaStream_t stream) {
  const SpecEntry& sp = spec_at(args.tb.specialization);
  if (sp.n_entities != args.cfg.n_entities || sp.n_items != args.cfg.n_items)
    return fail("specialization does not match the world (stale index?)%s");
  SpecArgs sa;
  sa.st = args.st;
  sa.joint_rot = args.tb.joint_rot;
  sa.mask = args.mask;
  sa.batch_dim = args.cfg.batch_dim;
  sa.use_mask = args.use_mask;
  sa.first_substep = args.first_substep;
  sa.n_substeps = args.n_substeps;
  sa.order = args.tb.env_order;
  sa.sig = args.tb.env_signature;
  sa.ent_params = args.ent_params;
  sa.ent_gravity = args.tb.ent_gravity;
  // tb.group selects the thread mapping of a specialised world: 1 = one thread per env,
  // VMAS_GROUP_TILE = a warp owns a tile of 32 envs and runs the narrow phase compacted
  if (args.tb.group == VMAS_GROUP_TILE) {
    if (!sp.has_tile) return fail("this specialization has no tile kernel (joints, or too many work items)%s");
    CUDA_OK(sp.launch_tile(sa, stream));
  } else
    CUDA_OK(sp.launch(sa, stream));
  return 1;
}

static int dispatch_step(const StepArgs& args, cudaStream_t stream) {
  if (args.tb.specialization >= 0) {
    if (args.tb.specialization >= num_specs()) return fail("specialization index out of range%s");
    return dispatch_spec(args, stream);
  }
  if (args.tb.group == 1) return dispatch_tpe(args, stream);
  if (args.tb.group == VMAS_GROUP_BLOCK) return launch_block(args, stream);
  const int G = args.tb.group, EPL = args.tb.ents_per_lane;
  if (G == 8 && EPL == 1) return launch_step<8, 1>(args, stream);
  if (G == 16 && EPL == 1) return launch_step<16, 1>(args, stream);
  if (G == 32 && EPL == 1) return launch_step<32, 1>(args, stream);
  if (G == 32 && EPL == 2) return launch_step<32, 2>(args, stream);
  if (G == 32 && EPL == 4) return launch_step<32, 4>(args, stream);
  return fail("unsupported lane layout (group, ents_per_lane)%s");
}

// ---- env scheduling: the envs of every 2048-env chunk sorted by their contact signature --------------
// Chunk-local on purpose: a global sort scatters a warp's 32 envs over the whole slab (measured: DRAM
// reads 2.3x the algorithmic bytes, the kernel turns memory-bound); within a chunk a warp's rows stay
// inside a 128 KB window per array that the chunk's 64 warps consume together.  The key is the raw
// signature (later = costlier items in the high bits), ties broken by env index: deterministic.
template <int ORDER_CHUNK>
__global__ void __launch_bounds__(ORDER_CHUNK / 2) order_sort_kernel(const uint32_t* __restrict__ sig, int B,
                                                                     int32_t* __restrict__ order) {
  constexpr int ORDER_THREADS = ORDER_CHUNK / 2;
  __shared__ unsigned long long key[ORDER_CHUNK];
  const long base = (long)blockIdx.x * ORDER_CHUNK;
  for (int i = threadIdx.x; i < ORDER_CHUNK; i += ORDER_THREADS)
    key[i] = base + i < B ? ((unsigned long long)sig[base + i] << 11) | (unsigned)i : ~0ull;  // padding sorts last
  __syncthreads();
  for (int k = 2; k <= ORDER_CHUNK; k <<= 1) {  // bitonic sort, ascending
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < ORDER_CHUNK; i += ORDER_THREADS) {
        const int partner = i ^ j;
        if (partner > i) {
          const unsigned long long a = key[i], b = key[partner];
          if ((a > b) == ((i & k) == 0)) {
            key[i] = b;
            key[partner] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < ORDER_CHUNK; i += ORDER_THREADS)
    if (base + i < B) order[base + i] = (int32_t)(base + (long)(key[i] & 2047u));
}

struct CopyArgs {
  VmasCopySegment seg[VMAS_MAX_COPY_SEGMENTS];
  int first_block[VMAS_MAX_COPY_SEGMENTS + 1];  // segment k is copied by blocks [first_block[k], first_block[k + 1])
};

// Every segment gets a share of the blocks in proportion to its size (an 8 MB observation block next to
// 128 KB reward rows); grid-stride inside the share; 16-byte words when both ends are 16-byte aligned.
__global__ void __launch_bounds__(256) copy_buffers_kernel(const CopyArgs a, const int n_segs) {
  int k = 0;
  while (k + 1 < n_segs && (int)blockIdx.x >= a.first_block[k + 1]) ++k;
  const VmasCopySegment s = a.seg[k];
  const size_t n_blocks = (size_t)(a.first_block[k + 1] - a.first_block[k]);
  const size_t tid = (size_t)(blockIdx.x - a.first_block[k]) * blockDim.x + threadIdx.x, stride = n_blocks * blockDim.x;
  const char* src = static_cast<const char*>(s.src);
  char* dst = static_cast<char*>(s.dst);
  size_t done = 0;
  if ((((uintptr_t)src | (uintptr_t)dst) & 15u) == 0) {
    const size_t words = s.bytes / 16;
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (size_t i = tid; i < words; i += stride) d4[i] = s4[i];
    done = words * 16;
  }
  for (size_t i = done + tid; i < s.bytes; i += stride) dst[i] = src[i];
}

struct CopyKinds {
  int32_t kind[VMAS_MAX_COPY_SEGMENTS];  // VMAS_DTYPE_F32: a byte copy; VMAS_DTYPE_F16 / _BF16: fp32 -> 16 bit
};

// fp32 [n] -> 16-bit [n], rounded to nearest even: the elements in front of the first 16-byte aligned source
// word one by one, then 16-byte loads and 8-byte stores (when the destination is 8-byte aligned there too; the
// two pointers advance 4 : 2 bytes per element, so that holds for all words or none), the tail one by one
template <int DT>
DEVI void convert_segment(const float* src, uint16_t* dst, const size_t n, const size_t tid, const size_t stride) {
  size_t head = (size_t)((16u - ((uintptr_t)src & 15u)) & 15u) / 4u;
  if (head > n) head = n;
  size_t done = n;
  if ((((uintptr_t)(dst + head)) & 7u) == 0) {
    const size_t words = (n - head) / 4;
    const float4* s4 = reinterpret_cast<const float4*>(src + head);
    uint2* d2 = reinterpret_cast<uint2*>(dst + head);
    for (size_t i = tid; i < words; i += stride) {
      const float4 v = s4[i];
      d2[i] = make_uint2(obs16x2_bits<DT>(v.x, v.y), obs16x2_bits<DT>(v.z, v.w));
    }
    for (size_t i = tid; i < head; i += stride) dst[i] = obs16_bits<DT>(src[i]);
    done = head + words * 4;
  } else {
    done = 0;
  }
  for (size_t i = done + tid; i < n; i += stride) dst[i] = obs16_bits<DT>(src[i]);
}

// copy_buffers_kernel with converting segments: the same split of the blocks over the segments
__global__ void __launch_bounds__(256) copy_convert_kernel(const CopyArgs a, const CopyKinds kinds, const int n_segs) {
  int k = 0;
  while (k + 1 < n_segs && (int)blockIdx.x >= a.first_block[k + 1]) ++k;
  const VmasCopySegment s = a.seg[k];
  const size_t n_blocks = (size_t)(a.first_block[k + 1] - a.first_block[k]);
  const size_t tid = (size_t)(blockIdx.x - a.first_block[k]) * blockDim.x + threadIdx.x, stride = n_blocks * blockDim.x;
  const int kind = kinds.kind[k];
  if (kind == VMAS_DTYPE_F16) {
    convert_segment<VMAS_DTYPE_F16>(static_cast<const float*>(s.src), static_cast<uint16_t*>(s.dst), s.bytes / 4, tid, stride);
    return;
  }
  if (kind == VMAS_DTYPE_BF16) {
    convert_segment<VMAS_DTYPE_BF16>(static_cast<const float*>(s.src), static_cast<uint16_t*>(s.dst), s.bytes / 4, tid, stride);
    return;
  }
  const char* src = static_cast<const char*>(s.src);
  char* dst = static_cast<char*>(s.dst);
  size_t done = 0;
  if ((((uintptr_t)src | (uintptr_t)dst) & 15u) == 0) {
    const size_t words = s.bytes / 16;
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (size_t i = tid; i < words; i += stride) d4[i] = s4[i];
    done = words * 16;
  }
  for (size_t i = done + tid; i < s.bytes; i += stride) dst[i] = src[i];
}

static int launch_broad_phase(const StepArgs& args, cudaStream_t stream) {
  const long blocks = ((long)args.cfg.batch_dim + 31) / 32;
  broad_phase_kernel<<<(unsigned)blocks, dim3(32, BROAD_SLICES), args.mask_words * sizeof(uint32_t), stream>>>(args);
  CUDA_OK(cudaGetLastError());
  return 1;
}

}  // namespace vmas

using namespace vmas;

extern "C" {

int vmas_b200_abi_version(void) { return VMAS_B200_ABI_VERSION; }

int vmas_b200_num_specializations(void) { return num_specs(); }

int vmas_b200_find_specialization(uint64_t world_hash) {
  for (int i = 0; i < num_specs(); ++i)
    if (spec_at(i).hash == world_hash) return i;
  return -1;
}

int vmas_b200_register_specialization(uint64_t world_hash, int32_t n_entities, int32_t n_items, void* launch,
                                      void* launch_tile, int32_t spec_args_bytes) {
  if (!launch) return fail("null launch function%s");
  if (spec_args_bytes != (int32_t)sizeof(SpecArgs)) return fail("SpecArgs layout mismatch: rebuild the specialisation%s");
  const int have = vmas_b200_find_specialization(world_hash);
  if (have >= 0) return have;
  if (g_num_dyn_specs >= VMAS_MAX_RUNTIME_SPECS) return fail("too many run-time specialisations%s");
  SpecEntry& e = g_dyn_specs[g_num_dyn_specs];
  e.hash = world_hash;
  e.name = "run-time specialisation";
  e.n_entities = n_entities;
  e.n_items = n_items;
  e.launch = reinterpret_cast<cudaError_t (*)(const SpecArgs&, cudaStream_t)>(launch);
  e.launch_tile = reinterpret_cast<cudaError_t (*)(const SpecArgs&, cudaStream_t)>(launch_tile);
  e.has_tile = launch_tile != nullptr;
  return kNumSpecs + g_num_dyn_specs++;
}

int vmas_b200_register_step_kernel(uint64_t key, int32_t n_entities, int32_t n_items, void* launch, void* launch_env,
                                   int32_t spec_args_bytes, int32_t epi_args_bytes, int32_t act_args_bytes) {
  if (!launch) return fail("null launch function%s");
  if (spec_args_bytes != (int32_t)sizeof(SpecArgs) || epi_args_bytes != (int32_t)sizeof(EpiArgs) ||
      (launch_env && act_args_bytes != (int32_t)sizeof(ActArgs)))
    return fail("SpecArgs / EpiArgs / ActArgs layout mismatch: rebuild the whole-step kernel%s");
  for (int i = 0; i < g_num_fused; ++i)
    if (g_fused[i].key == key) return i + 1;
  if (g_num_fused >= VMAS_MAX_RUNTIME_SPECS) return fail("too many whole-step kernels%s");
  FusedEntry& e = g_fused[g_num_fused];
  e.key = key;
  e.n_entities = n_entities;
  e.n_items = n_items;
  e.launch = reinterpret_cast<cudaError_t (*)(const SpecArgs&, const EpiArgs&, cudaStream_t)>(launch);
  e.launch_env =
      reinterpret_cast<cudaError_t (*)(const SpecArgs&, const EpiArgs&, const ActArgs&, cudaStream_t)>(launch_env);
  return ++g_num_fused;
}

int vmas_b200_specialization_has_tile(int index) {
  return (index >= 0 && index < num_specs() && spec_at(index).has_tile) ? 1 : 0;
}

const char* vmas_b200_specialization_name(int index) {
  return (index >= 0 && index < num_specs()) ? spec_at(index).name : "";
}

const char* vmas_b200_last_error(void) { return g_last_error; }

// `fused` > 0: the launches go to that whole-step kernel (its epilogue `epi` runs behind the last substep)
static int substeps_impl(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                         uint32_t* mask, int exact_broad_phase, int first_substep, int n_substeps,
                         void* cuda_stream, void* ev_begin, void* ev_end, int fused = 0,
                         const EpiArgs* epi = nullptr, const float* ent_params = nullptr) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (cfg->n_agents > 0 && (!st->force || !st->torque)) return fail("null force/torque pointer%s");
  if (cfg->n_items > 0 && (!tb->item_f32 || !tb->item_i32 || !tb->sched || !tb->inc || !tb->inc_off))
    return fail("null item tables%s");
  if (n_substeps <= 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  StepArgs args;
  args.cfg = *cfg;
  args.tb = *tb;
  args.st = *st;
  args.mask = mask;
  args.mask_words = (cfg->n_masked + 31) / 32;
  args.ent_params = ent_params;
  const bool masked = cfg->n_masked > 0 && exact_broad_phase;
  if (masked && (!mask || !tb->masked_items)) return fail("broad-phase mask scratch missing%s");
  int launches = 0;
  if (!masked) {
    args.use_mask = 0;
    args.first_substep = first_substep;
    args.n_substeps = n_substeps;
    if (ev_begin) CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(ev_begin), stream));
    int r = fused > 0 ? dispatch_fused(args, fused, *epi, stream) : dispatch_step(args, stream);
    if (r < 0) return r;
    if (ev_end) CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(ev_end), stream));
    return r;
  }
  args.use_mask = 1;
  for (int s = first_substep; s < first_substep + n_substeps; ++s) {
    args.first_substep = s;
    args.n_substeps = 1;
    int r = 0;
    if (!(exact_broad_phase == 2 && s == first_substep)) {  // 2: the caller's fused ingest launch built this mask
      r = launch_broad_phase(args, stream);
      if (r < 0) return r;
      launches += r;
    }
    if (ev_begin && s == first_substep) CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(ev_begin), stream));
    r = fused > 0 ? dispatch_fused(args, fused, *epi, stream) : dispatch_step(args, stream);
    if (r < 0) return r;
    launches += r;
  }
  if (ev_end) CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(ev_end), stream));
  return launches;
}

int vmas_b200_world_substeps(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                             uint32_t* mask, int exact_broad_phase, int first_substep, int n_substeps,
                             void* cuda_stream) {
  return substeps_impl(cfg, tb, st, mask, exact_broad_phase, first_substep, n_substeps, cuda_stream, nullptr,
                       nullptr);
}

int vmas_b200_world_step_timed(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                               uint32_t* mask, int exact_broad_phase, void* cuda_stream, void* ev_begin,
                               void* ev_end) {
  if (!cfg) return fail("null argument%s");
  return substeps_impl(cfg, tb, st, mask, exact_broad_phase, 0, cfg->substeps, cuda_stream, ev_begin, ev_end);
}

int vmas_b200_world_step_params(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const float* ent_params,
                                const VmasState* st, uint32_t* mask, int exact_broad_phase, void* cuda_stream) {
  if (!cfg) return fail("null argument%s");
  return substeps_impl(cfg, tb, st, mask, exact_broad_phase, 0, cfg->substeps, cuda_stream, nullptr, nullptr, 0,
                       nullptr, ent_params);
}

int vmas_b200_world_step(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                         uint32_t* mask, int exact_broad_phase, void* cuda_stream) {
  return vmas_b200_world_step_params(cfg, tb, nullptr, st, mask, exact_broad_phase, cuda_stream);
}

int vmas_b200_broad_phase(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                          uint32_t* mask, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (cfg->n_masked <= 0) return 0;
  if (!mask || !tb->masked_items) return fail("broad-phase mask scratch missing%s");
  StepArgs args;
  args.cfg = *cfg;
  args.tb = *tb;
  args.st = *st;
  args.mask = mask;
  args.mask_words = (cfg->n_masked + 31) / 32;
  args.use_mask = 1;
  args.first_substep = 0;
  args.n_substeps = 1;
  return launch_broad_phase(args, static_cast<cudaStream_t>(cuda_stream));
}

int vmas_b200_cast_rays(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                        int32_t src_entity, const int32_t* targets, int32_t n_targets,
                        const float* angles, int32_t n_rays, int32_t add_rot_of, float max_range,
                        float* out, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (!angles || !out || n_rays <= 0) return fail("bad ray buffers%s");
  if (src_entity < 0 || src_entity >= cfg->n_entities) return fail("source entity out of range%s");
  if (n_targets > 0 && !targets) return fail("null target list%s");
  RayArgs a;
  a.cfg = *cfg;
  a.tb = *tb;
  a.st = *st;
  a.targets = targets;
  a.angles = angles;
  a.out = out;
  a.src = src_entity;
  a.n_targets = n_targets;
  a.n_rays = n_rays;
  a.add_rot_of = add_rot_of;
  a.max_range = max_range;
  const int threads = 256;
  const long total = (long)cfg->batch_dim * n_rays;
  const long blocks = (total + threads - 1) / threads;
  cast_rays_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_pair_query(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                         int32_t a, int32_t b, int32_t mode, void* out, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (!out) return fail("null output%s");
  if (a < 0 || b < 0 || a >= cfg->n_entities || b >= cfg->n_entities) return fail("entity out of range%s");
  QueryArgs q;
  q.cfg = *cfg;
  q.tb = *tb;
  q.st = *st;
  q.a = a;
  q.b = b;
  q.mode = mode;
  q.point = nullptr;
  q.out = out;
  const int threads = 256;
  const long blocks = ((long)cfg->batch_dim + threads - 1) / threads;
  pair_query_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(q);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_point_query(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                          int32_t entity, const float* point, float* out, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (!out || !point) return fail("null buffer%s");
  if (entity < 0 || entity >= cfg->n_entities) return fail("entity out of range%s");
  QueryArgs q;
  q.cfg = *cfg;
  q.tb = *tb;
  q.st = *st;
  q.a = entity;
  q.b = entity;
  q.mode = 0;
  q.point = point;
  q.out = out;
  const int threads = 256;
  const long blocks = ((long)cfg->batch_dim + threads - 1) / threads;
  point_query_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(q);
  CUDA_OK(cudaGetLastError());
  return 1;
}

static int ingest_impl(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                       const VmasAgentActions* agents, int32_t n_agents, int32_t clamp, uint8_t* bad_flag, float* steps,
                       uint32_t* mask, void* cuda_stream);

int vmas_b200_ingest_actions(const VmasWorldConfig* cfg, const VmasState* st, const VmasAgentActions* agents,
                             int32_t n_agents, int32_t clamp, uint8_t* bad_flag, float* steps, void* cuda_stream) {
  return ingest_impl(cfg, nullptr, st, agents, n_agents, clamp, bad_flag, steps, nullptr, cuda_stream);
}

int vmas_b200_ingest_actions_broad_phase(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                         const VmasAgentActions* agents, int32_t n_agents, int32_t clamp,
                                         uint8_t* bad_flag, float* steps, uint32_t* mask, void* cuda_stream) {
  if (!tb || !mask) return fail("null argument%s");
  return ingest_impl(cfg, tb, st, agents, n_agents, clamp, bad_flag, steps, mask, cuda_stream);
}

static int ingest_impl(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                       const VmasAgentActions* agents, int32_t n_agents, int32_t clamp, uint8_t* bad_flag, float* steps,
                       uint32_t* mask, void* cuda_stream) {
  if (!cfg || !st || !agents) return fail("null argument%s");
  if (n_agents <= 0 || n_agents > VMAS_MAX_INGEST_AGENTS) return fail("1..16 agents per ingest call%s");
  IngestArgs a;
  for (int i = 0; i < n_agents; ++i) {
    a.ag[i] = agents[i];
    if (!agents[i].actions || !agents[i].u) return fail("null action buffer%s");
    if (agents[i].action_size < 0 || agents[i].action_size > VMAS_MAX_ACTION_SIZE) return fail("action size > 8%s");
    if (agents[i].dynamics >= 0) {
      static const int need[] = {2, 3, 1, 1, 2, 2, 4};
      if (agents[i].dynamics > VMAS_DYN_DRONE) return fail("unknown dynamics code%s");
      if (!st->force || !st->torque) return fail("null force/torque pointer%s");
      if (agents[i].agent_index < 0 || agents[i].agent_index >= cfg->n_agents) return fail("agent index%s");
      if (agents[i].action_size < need[agents[i].dynamics]) return fail("action too small for dynamics%s");
      if (agents[i].dynamics >= VMAS_DYN_FORWARD && agents[i].dynamics != VMAS_DYN_ROTATION) {
        if (agents[i].entity_index < 0 || agents[i].entity_index >= cfg->n_entities) return fail("entity index%s");
        if (!st->pos || !st->vel || !st->rot || !st->ang_vel) return fail("null state pointer%s");
      }
      if (agents[i].dynamics == VMAS_DYN_DRONE && !agents[i].dyn_state) return fail("drone without its state buffer%s");
    }
  }
  a.st = *st;
  a.bad_flag = bad_flag;
  a.steps = steps;
  a.n_entities = cfg->n_entities;
  a.n_agents_total = cfg->n_agents;
  a.n = n_agents;
  a.batch_dim = cfg->batch_dim;
  a.clamp = clamp;
  const int threads = 256;
  const long total = (long)cfg->batch_dim * n_agents;
  const unsigned n_ingest = (unsigned)((total + threads - 1) / threads);
  bool kinematic = false;
  for (int i = 0; i < n_agents; ++i) kinematic |= agents[i].dynamics >= VMAS_DYN_DIFF_DRIVE;
  if (mask && cfg->n_masked > 0) {
    if (!tb->masked_items || !tb->item_i32 || !tb->item_f32 || !st->pos) return fail("null broad-phase tables%s");
    StepArgs sa;
    sa.cfg = *cfg;
    sa.tb = *tb;
    sa.st = *st;
    sa.mask = mask;
    sa.mask_words = (cfg->n_masked + 31) / 32;
    sa.use_mask = 1;
    sa.first_substep = 0;
    sa.n_substeps = 1;
    const unsigned n_broad = (unsigned)(((long)cfg->batch_dim + 31) / 32);
    const dim3 block(32, BROAD_SLICES);
    const size_t smem = sa.mask_words * sizeof(uint32_t);
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (kinematic)
      ingest_broad_kernel<true><<<n_ingest + n_broad, block, smem, stream>>>(a, sa, (int)n_ingest);
    else
      ingest_broad_kernel<false><<<n_ingest + n_broad, block, smem, stream>>>(a, sa, (int)n_ingest);
  } else if (kinematic) {
    ingest_actions_kernel<true><<<n_ingest, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  } else {
    ingest_actions_kernel<false><<<n_ingest, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  }
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_velocity_controller(const VmasWorldConfig* cfg, const VmasState* st, int32_t entity, float* u,
                                  float* accum, float* prev, float gain, float inv_ti, float td, float dt,
                                  float windup, float mass, void* cuda_stream) {
  if (!cfg || !st || !st->vel || !u || !accum || !prev) return fail("null argument%s");
  if (entity < 0 || entity >= cfg->n_entities) return fail("entity index%s");
  if (cfg->batch_dim <= 0 || !(dt > 0.f)) return fail("empty batch or dt <= 0%s");
  PidArgs a;
  a.vel = st->vel;
  a.u = u;
  a.accum = accum;
  a.prev = prev;
  a.entity = entity;
  a.n_entities = cfg->n_entities;
  a.batch_dim = cfg->batch_dim;
  a.gain = gain;
  a.inv_ti = inv_ti;
  a.td = td;
  a.dt = dt;
  a.windup = windup;
  a.mass = mass;
  const int threads = 256;
  const long total = (long)cfg->batch_dim * 2;
  velocity_controller_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0,
                               static_cast<cudaStream_t>(cuda_stream)>>>(a);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_cast_rays_batched(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                int32_t n_sensors, const int32_t* src, const int32_t* target_off,
                                const int32_t* targets, const float* angles, const float* max_range,
                                int32_t n_rays, float* out, const int64_t* out_offsets, int64_t out_env_stride,
                                int32_t flags, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (out_env_stride != 0 && out_env_stride < n_rays) return fail("out_env_stride < n_rays%s");
  if (n_sensors <= 0 || n_rays <= 0) return fail("empty sensor batch%s");
  if (!src || !target_off || !angles || !max_range || !out) return fail("null sensor buffer%s");
  RayBatchArgs a;
  a.base.cfg = *cfg;
  a.base.tb = *tb;
  a.base.st = *st;
  a.base.targets = nullptr;
  a.base.angles = angles;
  a.base.out = out;
  a.base.src = 0;
  a.base.n_targets = 0;
  a.base.n_rays = n_rays;
  a.base.add_rot_of = 0;
  a.base.max_range = 0.f;
  a.src = src;
  a.target_off = target_off;
  a.all_targets = targets;
  a.range = max_range;
  a.out_off = out_offsets;
  a.out_env_stride = out_env_stride ? out_env_stride : n_rays;
  a.n_sensors = n_sensors;
  a.flags = flags;
  if (n_sensors > 65535) return fail("more than 65535 sensors in one batch%s");
  const unsigned bx = (unsigned)(n_rays < 256 ? n_rays : 256), by = 256 / bx;
  const dim3 block(bx, by);
  const dim3 grid((unsigned)((cfg->batch_dim + by - 1) / by), (unsigned)n_sensors);
  const size_t smem = by * RAY_MASK_WORDS * sizeof(uint32_t);
  if (flags & VMAS_RAYS_SPHERE_TARGETS) {
    cast_rays_batched_kernel<true><<<grid, block, smem, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  } else {
    cast_rays_batched_kernel<false><<<grid, block, smem, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  }
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_gather_observations(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* columns,
                                  int32_t n_rows, int32_t width, float* out, void* cuda_stream) {
  return vmas_b200_gather_observations_buffers(cfg, st, columns, n_rows, width, out, nullptr, 0, cuda_stream);
}

int vmas_b200_gather_observations_buffers(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* columns,
                                          int32_t n_rows, int32_t width, float* out, const float* const* buffers,
                                          int32_t n_buffers, void* cuda_stream) {
  if (!cfg || !st || !columns || !out) return fail("null argument%s");
  if (n_buffers < 0 || n_buffers > VMAS_OBS_MAX_BUFFERS || (n_buffers > 0 && !buffers)) return fail("0..8 observation buffers%s");
  if (!st->pos || !st->vel || !st->rot || !st->ang_vel) return fail("null state pointer%s");
  if (n_rows <= 0 || width <= 0 || cfg->batch_dim <= 0) return fail("empty observation block%s");
  ObsArgs a;
  a.st = *st;
  a.cols = columns;
  a.out = out;
  a.rows = n_rows;
  a.width = width;
  a.batch_dim = cfg->batch_dim;
  a.n_entities = cfg->n_entities;
  for (int i = 0; i < VMAS_OBS_MAX_BUFFERS; ++i) a.buffers[i] = i < n_buffers ? buffers[i] : nullptr;
  for (int i = 0; i < n_buffers; ++i)
    if (!buffers[i]) return fail("null observation buffer%s");
  if (n_rows > 65535) return fail("more than 65535 observation rows%s");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  // vector width: the widest that divides the row (and keeps every store aligned)
  const int vec = (width % 4 == 0 && ((uintptr_t)out % 16 == 0)) ? 4 : (width % 2 == 0 && ((uintptr_t)out % 8 == 0)) ? 2 : 1;
  const int groups = width / vec;
  if (groups > 256) return fail("observation rows wider than 1024 columns are not supported%s");
  const unsigned bx = (unsigned)groups, by = 256 / bx;
  const dim3 block(bx, by);
  int tile = 0;
  size_t smem = 0;
  if (obs_tile(cfg->n_entities, &tile, &smem) < 0) return -1;
  const dim3 grid((unsigned)((cfg->batch_dim + tile - 1) / tile), (unsigned)n_rows);
  auto kern = vec == 4 ? gather_observations_kernel<4> : vec == 2 ? gather_observations_kernel<2> : gather_observations_kernel<1>;
  if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, block, smem, stream>>>(a, tile);
  CUDA_OK(cudaGetLastError());
  return 1;
}

}  // extern "C"

template <int VEC>
static auto post_step_kernel_of(int obs_dtype) {
  return obs_dtype == VMAS_DTYPE_F16 ? post_step_kernel<VEC, VMAS_DTYPE_F16>
         : obs_dtype == VMAS_DTYPE_BF16 ? post_step_kernel<VEC, VMAS_DTYPE_BF16>
                                        : post_step_kernel<VEC, VMAS_DTYPE_F32>;
}

// vmas_b200_post_step with the observation rows stored as `obs_dtype` (VMAS_DTYPE_*)
static int post_step_impl(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                          const VmasStepProgram* program, const int32_t* columns, int32_t n_rows, int32_t width,
                          void* obs_out, int obs_dtype, void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (obs_dtype < VMAS_DTYPE_F32 || obs_dtype > VMAS_DTYPE_BF16) return fail("unknown observation dtype%s");
  const bool has_prog = program && program->n_instr > 0, has_obs = columns && n_rows > 0;
  if (!has_prog && !has_obs) return fail("neither a program nor observation rows%s");
  if (has_prog && (program->n_instr > VMAS_PROG_MAX_INSTR)) return fail("program too long%s");
  if (has_obs && (!obs_out || width <= 0 || n_rows > 65534)) return fail("bad observation block%s");
  ProgArgs pa;
  pa.base.cfg = *cfg;
  pa.base.tb = *tb;
  pa.base.st = *st;
  pa.base.a = pa.base.b = pa.base.mode = 0;
  pa.base.point = nullptr;
  pa.base.out = nullptr;
  pa.prog.n_instr = 0;
  if (has_prog) {
    pa.prog = *program;
    for (int i = 0; i < program->n_instr; ++i) {
      const VmasProgInstr& in = program->instr[i];
      if (in.dst >= VMAS_PROG_REGS || in.a >= VMAS_PROG_REGS && in.op >= VMAS_OP_ADD && in.op <= VMAS_OP_WHERE)
        return fail("program register out of range%s");
      if (in.op == VMAS_OP_SHAPING && in.dst + 1 >= VMAS_PROG_REGS) return fail("program register out of range%s");
    }
  }
  ObsArgs oa;
  oa.st = *st;
  oa.cols = columns;
  oa.out = obs_out;
  oa.rows = has_obs ? n_rows : 0;
  oa.width = has_obs ? width : 4;
  oa.batch_dim = cfg->batch_dim;
  oa.n_entities = cfg->n_entities;
  for (int i = 0; i < VMAS_OBS_MAX_BUFFERS; ++i) oa.buffers[i] = nullptr;  // (buffer columns need a launch of their own)
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  int vec = 4;
  if (has_obs) {
    // 16-bit rows: the same groups of columns, stores of half the size
    const uintptr_t a16 = obs_dtype == VMAS_DTYPE_F32 ? 16 : 8, a8 = obs_dtype == VMAS_DTYPE_F32 ? 8 : 4;
    vec = (width % 4 == 0 && ((uintptr_t)obs_out % a16 == 0)) ? 4 : (width % 2 == 0 && ((uintptr_t)obs_out % a8 == 0)) ? 2 : 1;
  }
  const int groups = oa.width / vec;
  if (groups > 256 || groups < 1) return fail("observation rows wider than 1024 columns are not supported%s");
  const unsigned bx = (unsigned)groups, by = 256 / bx;
  const dim3 block(bx, by);
  int tile = 0;
  size_t smem = 0;
  if (obs_tile(cfg->n_entities, &tile, &smem) < 0) return -1;
  const dim3 grid((unsigned)((cfg->batch_dim + tile - 1) / tile), (unsigned)(oa.rows + (has_prog ? 1 : 0)));
  auto kern = vec == 4 ? post_step_kernel_of<4>(obs_dtype) : vec == 2 ? post_step_kernel_of<2>(obs_dtype) : post_step_kernel_of<1>(obs_dtype);
  if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, block, smem, stream>>>(oa, tile, pa);
  CUDA_OK(cudaGetLastError());
  return 1;
}

extern "C" {

int vmas_b200_post_step(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                        const VmasStepProgram* program, const int32_t* columns, int32_t n_rows, int32_t width,
                        float* obs_out, void* cuda_stream) {
  return post_step_impl(cfg, tb, st, program, columns, n_rows, width, obs_out, VMAS_DTYPE_F32, cuda_stream);
}

int vmas_b200_pair_query_batched(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                 const int32_t* pairs, int32_t n_pairs, int32_t mode, void* out,
                                 void* cuda_stream) {
  if (check_common(cfg, tb, st) < 0) return -1;
  if (!pairs || !out || n_pairs <= 0) return fail("bad pair batch%s");
  const bool spheres = mode & VMAS_QUERY_SPHERES;
  mode &= ~VMAS_QUERY_SPHERES;
  if (mode < 0 || mode > 2) return fail("unknown pair query mode%s");
  PairBatchArgs a;
  a.base.cfg = *cfg;
  a.base.tb = *tb;
  a.base.st = *st;
  a.base.a = a.base.b = 0;
  a.base.mode = mode;
  a.base.point = nullptr;
  a.base.out = out;
  a.pairs = pairs;
  a.n_pairs = n_pairs;
  const int threads = 128;
  a.chunk = pairs_per_thread(cfg->batch_dim, n_pairs);
  const int chunks = (n_pairs + a.chunk - 1) / a.chunk;
  if (chunks > 65535) return fail("too many pairs in one batch%s");
  const dim3 grid((unsigned)((cfg->batch_dim + threads - 1) / threads), (unsigned)chunks);
  if (spheres) {
    pair_query_spheres_kernel<<<grid, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  } else {
    pair_query_batched_kernel<<<grid, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  }
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_distance_shaping(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* pairs,
                               int32_t n_pairs, float factor, float* prev, float* dist, float* rew,
                               void* cuda_stream) {
  if (!cfg || !st || !st->pos || !pairs || !prev || !rew) return fail("null argument%s");
  if (n_pairs <= 0 || cfg->batch_dim <= 0) return fail("empty pair batch%s");
  ShapingArgs a;
  a.pos = st->pos;
  a.pairs = pairs;
  a.prev = prev;
  a.dist = dist;
  a.rew = rew;
  a.factor = factor;
  a.n_pairs = n_pairs;
  a.n_entities = cfg->n_entities;
  a.batch_dim = cfg->batch_dim;
  const int threads = 128;
  a.chunk = pairs_per_thread(cfg->batch_dim, n_pairs);
  const int chunks = (n_pairs + a.chunk - 1) / a.chunk;
  if (chunks > 65535) return fail("too many pairs in one batch%s");
  const dim3 grid((unsigned)((cfg->batch_dim + threads - 1) / threads), (unsigned)chunks);
  distance_shaping_kernel<<<grid, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_build_env_order(const uint32_t* signature, int32_t batch_dim, int32_t* order, int32_t chunk,
                              void* cuda_stream) {
  if (!signature || !order) return fail("null argument%s");
  if (batch_dim <= 0) return fail("empty batch%s");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const int blocks = (int)(((size_t)batch_dim + chunk - 1) / (chunk > 0 ? chunk : 1));
  switch (chunk) {
    case 256: order_sort_kernel<256><<<blocks, 128, 0, stream>>>(signature, batch_dim, order); break;
    case 512: order_sort_kernel<512><<<blocks, 256, 0, stream>>>(signature, batch_dim, order); break;
    case 1024: order_sort_kernel<1024><<<blocks, 512, 0, stream>>>(signature, batch_dim, order); break;
    case 2048: order_sort_kernel<2048><<<blocks, 1024, 0, stream>>>(signature, batch_dim, order); break;
    default: return fail("env order chunk must be 256, 512, 1024 or 2048%s");
  }
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_set_l2_fetch_granularity(int32_t bytes) {
  // 32, 64 or 128: how much the L2 fetches from DRAM on a sector miss (a device-wide hint)
  CUDA_OK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)bytes));
  size_t got = 0;
  CUDA_OK(cudaDeviceGetLimit(&got, cudaLimitMaxL2FetchGranularity));
  return (int)got;
}

// ---- hand-out copy of a step's packed outputs ---------------------------------------------------
// Environment.step in CUDA-graph mode hands out fresh copies of the buffers the graph writes.  One
// kernel for all of them: cudaMemcpyAsync D2D runs on a copy engine, where it queues behind a
// concurrent device->host download of the previous step's results (measured: the pipelined e2e loop
// serialised completely); an SM copy does not.
int vmas_b200_copy_buffers(const VmasCopySegment* segs, int32_t n_segs, void* cuda_stream) {
  if (!segs || n_segs <= 0 || n_segs > VMAS_MAX_COPY_SEGMENTS) return fail("1..VMAS_MAX_COPY_SEGMENTS segments expected%s");
  CopyArgs a;
  const int threads = 256;
  const size_t per_block = (size_t)threads * 4 * 16;  // ~4 x 16 B per thread
  int blocks = 0;
  for (int i = 0; i < n_segs; ++i) {
    if (!segs[i].src || !segs[i].dst) return fail("null copy segment%s");
    a.seg[i] = segs[i];
    a.first_block[i] = blocks;
    size_t want = (segs[i].bytes + per_block - 1) / per_block;
    want = want < 1 ? 1 : (want > 132 * 8 ? 132 * 8 : want);  // at most 8 blocks per SM of an H100 SXM
    blocks += (int)want;
  }
  a.first_block[n_segs] = blocks;
  copy_buffers_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a, n_segs);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_copy_buffers_convert(const VmasCopySegment* segs, const int32_t* kinds, int32_t n_segs,
                                   void* cuda_stream) {
  if (!segs || !kinds || n_segs <= 0 || n_segs > VMAS_MAX_COPY_SEGMENTS) return fail("1..VMAS_MAX_COPY_SEGMENTS segments expected%s");
  CopyArgs a;
  CopyKinds k;
  const int threads = 256;
  const size_t per_block = (size_t)threads * 4 * 16;  // ~4 x 16 B (of the source) per thread
  int blocks = 0;
  for (int i = 0; i < n_segs; ++i) {
    if (!segs[i].src || !segs[i].dst) return fail("null copy segment%s");
    if (kinds[i] < VMAS_DTYPE_F32 || kinds[i] > VMAS_DTYPE_BF16) return fail("unknown copy segment kind%s");
    if (kinds[i] != VMAS_DTYPE_F32 &&
        (segs[i].bytes % 4 || ((uintptr_t)segs[i].src & 3u) || ((uintptr_t)segs[i].dst & 1u)))
      return fail("a converting segment needs whole fp32 values at 4-byte aligned sources, 2-byte aligned destinations%s");
    a.seg[i] = segs[i];
    k.kind[i] = kinds[i];
    a.first_block[i] = blocks;
    size_t want = (segs[i].bytes + per_block - 1) / per_block;
    want = want < 1 ? 1 : (want > 132 * 8 ? 132 * 8 : want);  // at most 8 blocks per SM of an H100 SXM
    blocks += (int)want;
  }
  a.first_block[n_segs] = blocks;
  copy_convert_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(a, k, n_segs);
  CUDA_OK(cudaGetLastError());
  return 1;
}

int vmas_b200_graph_num_nodes(void* cuda_graph) {
  if (!cuda_graph) return fail("null graph%s");
  size_t n = 0;
  CUDA_OK(cudaGraphGetNodes(static_cast<cudaGraph_t>(cuda_graph), nullptr, &n));
  return (int)n;
}

// ---- Environment.step as one call ------------------------------------------------------------------------
// The host side of a step is otherwise three crossings of the FFI (ingest, graph replay through torch,
// hand-out copy) with their marshalling — more host time than the kernels take.

// where this step's post stage writes: the caller's static buffers, or (direct mode) this step's fresh blocks
struct StepTargets {
  void* obs_out;
  int obs_dtype;  // of obs_out: s->obs_dtype in the caller's fresh block, fp32 in the static buffer
  const VmasStepProgram* program;
  VmasStepProgram patched;
};

static int env_step_targets(const VmasEnvStep* s, StepTargets& t) {
  t.obs_out = s->obs_out;
  t.obs_dtype = VMAS_DTYPE_F32;
  t.program = s->program;
  if (s->obs_dtype < VMAS_DTYPE_F32 || s->obs_dtype > VMAS_DTYPE_BF16) return fail("unknown observation dtype%s");
  if (s->obs_block >= 0 && s->columns && s->n_rows > 0) {
    if (s->obs_block >= s->n_out_blocks || !s->out_blocks[s->obs_block]) return fail("observation rows without their block%s");
    t.obs_out = static_cast<char*>(s->out_blocks[s->obs_block]) + s->obs_offset;
    t.obs_dtype = s->obs_dtype;
  }
  if (s->n_mirrors > 0) {
    if (!s->program || s->n_mirrors > VMAS_PROG_MAX_BUFFERS) return fail("mirrored stores without a program%s");
    t.patched = *s->program;
    for (int i = 0; i < s->n_mirrors; ++i) {
      const int slot = s->mirror_slot[i], b = s->mirror_block[i];
      if (slot < 0 || slot >= VMAS_PROG_MAX_BUFFERS || b < 0 || b >= s->n_out_blocks || !s->out_blocks[b])
        return fail("bad mirrored store%s");
      t.patched.buffers[slot] = static_cast<char*>(s->out_blocks[b]) + s->mirror_offset[i];
    }
    t.program = &t.patched;
  }
  if (s->columns && s->n_rows > 0 && (!t.obs_out || ((uintptr_t)t.obs_out & 15u)))
    return fail("observation block missing or not 16-byte aligned%s");
  return 0;
}

static int env_step_hand_out(const VmasEnvStep* s, void* cuda_stream) {
  if (s->n_segs <= 0) return 0;
  if (s->n_segs > VMAS_MAX_COPY_SEGMENTS || !s->segs || !s->seg_block) return fail("bad hand-out segments%s");
  VmasCopySegment segs[VMAS_MAX_COPY_SEGMENTS];
  for (int i = 0; i < s->n_segs; ++i) {
    const int b = s->seg_block[i];
    if (b < 0 || b >= s->n_out_blocks || !s->out_blocks[b]) return fail("hand-out segment without its block%s");
    segs[i].src = s->segs[i].src;
    segs[i].dst = static_cast<char*>(s->out_blocks[b]) + reinterpret_cast<uintptr_t>(s->segs[i].dst);
    segs[i].bytes = s->segs[i].bytes;
  }
  if (s->seg_kind) return vmas_b200_copy_buffers_convert(segs, s->seg_kind, s->n_segs, cuda_stream);
  return vmas_b200_copy_buffers(segs, s->n_segs, cuda_stream);
}

static EpiArgs epi_args_of(const StepTargets& t) {
  EpiArgs epi;
  epi.obs_out = t.obs_out;
  for (int i = 0; i < VMAS_PROG_MAX_BUFFERS; ++i) epi.buffers[i] = t.program ? t.program->buffers[i] : nullptr;
  return epi;
}

// The whole step as ONE launch (step_env_kernel).  1: launched; 0: not applicable this time (the batch does
// not fit the GPU at once, which the kernel's grid-wide barrier needs); < 0: error.
static int env_step_one_kernel(const VmasEnvStep* s, const StepTargets& t, cudaStream_t stream) {
  if (s->fused_kernel < 1 || s->fused_kernel > g_num_fused) return fail("unknown whole-step kernel%s");
  const FusedEntry& f = g_fused[s->fused_kernel - 1];
  if (!f.launch_env) return 0;
  if (check_common(s->cfg, s->tb, s->st) < 0) return -1;
  if (f.n_entities != s->cfg->n_entities || f.n_items != s->cfg->n_items)
    return fail("whole-step kernel does not match the world (stale handle?)%s");
  if (!s->st->force || !s->st->torque || !s->agents) return fail("null force/torque/agents pointer%s");
  const bool masked = s->cfg->n_masked > 0 && s->exact_broad_phase;
  if (masked && !s->mask) return 0;  // (mask scratch: substeps x (mask words + 2) uint32, see VmasEnvStep)
  StepArgs args;
  args.cfg = *s->cfg;
  args.tb = *s->tb;
  args.st = *s->st;
  args.mask = s->mask;
  args.mask_words = (s->cfg->n_masked + 31) / 32;
  args.use_mask = masked ? 1 : 0;
  args.first_substep = 0;
  args.n_substeps = s->cfg->substeps;
  ActArgs act;
  if (s->n_agents > VMAS_MAX_INGEST_AGENTS) return 0;
  for (int i = 0; i < VMAS_MAX_INGEST_AGENTS; ++i) act.kind[i] = act.dyn[i] = act.size[i] = -1;  // (no tensor)
  for (int i = 0; i < s->n_agents; ++i) {
    const VmasAgentActions& ag = s->agents[i];
    if (!ag.actions || !ag.u) return fail("null action buffer%s");
    if (ag.action_size < 1 || ag.action_size > 4) return 0;
    // holonomic agents with 2 components: fp32 [B, 2] and int64 [B, 1] rows are read as 8-byte words, int64
    // [B, 2] rows as 16-byte words; other models read their [B, 1..4] rows one element at a time
    const bool lean = ag.dynamics == VMAS_DYN_HOLONOMIC && ag.action_size == 2;
    const uintptr_t align = !lean ? (ag.action_kind == VMAS_ACT_CONTINUOUS ? 3u : 7u)
                                  : ag.action_kind == VMAS_ACT_MULTIDISCRETE ? 15u : 7u;
    if (ag.action_kind != VMAS_ACT_CONTINUOUS && ag.action_kind != VMAS_ACT_DISCRETE &&
        ag.action_kind != VMAS_ACT_MULTIDISCRETE)
      return 0;
    if (((uintptr_t)ag.actions & align) || ((uintptr_t)ag.u & (lean ? 7u : 3u))) return 0;
    act.actions[i] = ag.actions;
    act.u[i] = ag.u;
    act.kind[i] = ag.action_kind;
    act.dyn[i] = ag.dynamics;
    act.size[i] = ag.action_size;
  }
  act.bad_flag = s->bad_flag;
  act.steps = s->steps;
  act.clamp = s->clamp;
  const cudaError_t err = f.launch_env(spec_args_of(args), epi_args_of(t), act, stream);
  if (err == cudaErrorCooperativeLaunchTooLarge || err == cudaErrorInvalidValue) {
    cudaGetLastError();  // (not an error of this call: the step goes out as separate launches)
    return 0;
  }
  CUDA_OK(err);
  return 1;
}

int vmas_b200_env_step(const VmasEnvStep* s, void* cuda_stream) {
  if (!s || !s->cfg || !s->tb || !s->st) return fail("null argument%s");
  if (s->n_out_blocks < 0 || s->n_out_blocks > VMAS_MAX_OUT_BLOCKS) return fail("too many output blocks%s");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  int launches = 0, r;
  StepTargets t;
  if (!s->graph_exec && env_step_targets(s, t) < 0) return -1;
  bool stepped = false;
  if (s->ingest_in_kernel && s->n_agents > 0 && s->fused_kernel > 0 && !s->graph_exec) {
    r = env_step_one_kernel(s, t, stream);
    if (r < 0) return r;
    launches += r;
    stepped = r > 0;
  }
  if (!stepped) {
    if (s->n_agents > 0) {
      r = ingest_impl(s->cfg, s->tb, s->st, s->agents, s->n_agents, s->clamp, s->bad_flag, s->steps, s->ingest_mask,
                      cuda_stream);
      if (r < 0) return r;
      launches += r;
    }
    if (s->graph_exec) {
      CUDA_OK(cudaGraphLaunch(static_cast<cudaGraphExec_t>(s->graph_exec), stream));
    } else {
      const bool has_post = (t.program && t.program->n_instr > 0) || (s->columns && s->n_rows > 0);
      if (s->fused_kernel > 0 && has_post) {
        // the whole-step kernel: the program and the observation rows run in the substep kernel's epilogue
        const EpiArgs epi = epi_args_of(t);
        r = substeps_impl(s->cfg, s->tb, s->st, s->mask, s->exact_broad_phase, 0, s->cfg->substeps, cuda_stream,
                          nullptr, nullptr, s->fused_kernel, &epi);
        if (r < 0) return r;
        launches += r;
      } else {
        r = substeps_impl(s->cfg, s->tb, s->st, s->mask, s->exact_broad_phase, 0, s->cfg->substeps, cuda_stream,
                          nullptr, nullptr);
        if (r < 0) return r;
        launches += r;
        if (has_post) {
          r = post_step_impl(s->cfg, s->tb, s->st, t.program, s->columns, s->n_rows, s->width, t.obs_out, t.obs_dtype,
                             cuda_stream);
          if (r < 0) return r;
          launches += r;
        }
      }
    }
  }
  r = env_step_hand_out(s, cuda_stream);
  if (r < 0) return r;
  return launches + r;
}

}  // extern "C"

#include "reset.cuh"  // device-side episode reset: vmas_b200_reset_state, vmas_b200_spawn_entities
