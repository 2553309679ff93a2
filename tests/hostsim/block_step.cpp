// block_step.cpp — TEST INFRASTRUCTURE: runs the generic substep phases of csrc/generic_step.cuh on the
// CPU (g++, shim/cuda_runtime.h) in two formulations, so the block-per-env kernel's ownership, barriers
// and accumulation order can be checked bit for bit without a GPU.  Not product code.
//   variant 0: the thread-per-env formulation — entities, then the work items in item order
//              (item_accumulate), then the entities again, one env after the other;
//   variant 1: step_block_kernel's — the block's threads one after the other between barriers, thread t
//              owning entities t, t + BLOCK, ...; phase B walks each entity's incidence list
//              (entity_accumulate).  The env's shared memory is poisoned with NaN first, so a field read
//              before its owner wrote it shows up.
#include <stdint.h>

#include <vector>

#include <cuda_runtime.h>
struct int4 {
  int x, y, z, w;
};
template <class T>
static inline T __ldg(const T* p) {
  return *p;
}

#include "generic_step.cuh"

using namespace vmas;

static constexpr int BLOCK = 128;  // STEP_BLOCK_THREADS

extern "C" {

int hostsim_generic_step(int variant, const VmasWorldConfig* cfg, const VmasPlanTables* tb, float* pos, float* vel,
                         float* rot, float* ang_vel, float* force, float* torque, const float* ent_params,
                         const uint32_t* mask, int use_mask, int first_substep, int n_substeps) {
  StepArgs a;
  a.cfg = *cfg;
  a.tb = *tb;
  a.st.pos = pos; a.st.vel = vel; a.st.rot = rot; a.st.ang_vel = ang_vel; a.st.force = force; a.st.torque = torque;
  a.mask = nullptr;
  a.use_mask = use_mask;
  a.mask_words = (cfg->n_masked + 31) / 32;
  a.first_substep = first_substep;
  a.n_substeps = n_substeps;
  a.ent_params = ent_params;
  const int E = cfg->n_entities, A = cfg->n_agents, NI = cfg->n_items;
  std::vector<float> sm((size_t)T_NF * E + a.mask_words + 1);
  float* col = sm.data();
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(sm.data() + (size_t)T_NF * E);
  EnvShared<1> sh;
  sh.pitch = 1;
  sh.px = col + (size_t)T_PX * E;
  sh.py = col + (size_t)T_PY * E;
  sh.rot = col + (size_t)T_ROT * E;
  sh.c = col + (size_t)T_C * E;
  sh.s = col + (size_t)T_S * E;
  sh.c2 = col + (size_t)T_C2 * E;
  sh.s2 = col + (size_t)T_S2 * E;
  sh.rfx = sh.rfy = sh.rta = sh.rtb = nullptr;
  const float sub_dt = cfg->sub_dt;
  for (long env = 0; env < cfg->batch_dim; ++env) {
    for (float& v : sm) v = NAN;
    if (use_mask)
      for (int w = 0; w < a.mask_words; ++w) s_mask[w] = mask[w];
    const size_t ebase = (size_t)env * E, abase = (size_t)env * A;
    if (variant == 0) {
      for (int e = 0; e < E; ++e) entity_load<1>(a, col, E, e, ebase);
      for (int sub = first_substep; sub < first_substep + n_substeps; ++sub) {
        for (int e = 0; e < E; ++e) entity_forces<1>(a, col, E, e, env, ebase, abase, sub_dt);
        for (int item = 0; item < NI; ++item) item_accumulate(a, sh, col, E, item, env, s_mask);
        for (int e = 0; e < E; ++e) entity_integrate<1>(a, col, E, e, env, sub, sub_dt);
      }
      for (int e = 0; e < E; ++e) entity_store<1>(a, col, E, e, ebase);
    } else {
      // every `for (t ...)` below is the block's threads between two __syncthreads()
      for (int t = 0; t < BLOCK; ++t)
        for (int e = t; e < E; e += BLOCK) entity_load<1>(a, col, E, e, ebase);
      for (int sub = first_substep; sub < first_substep + n_substeps; ++sub) {
        for (int t = 0; t < BLOCK; ++t)
          for (int e = t; e < E; e += BLOCK) entity_forces<1>(a, col, E, e, env, ebase, abase, sub_dt);
        for (int t = 0; t < BLOCK; ++t)
          for (int e = t; e < E; e += BLOCK) entity_accumulate(a, sh, col, E, e, env, s_mask);
        for (int t = 0; t < BLOCK; ++t)
          for (int e = t; e < E; e += BLOCK) entity_integrate<1>(a, col, E, e, env, sub, sub_dt);
      }
      for (int t = 0; t < BLOCK; ++t)
        for (int e = t; e < E; e += BLOCK) entity_store<1>(a, col, E, e, ebase);
    }
  }
  return 0;
}

}  // extern "C"
