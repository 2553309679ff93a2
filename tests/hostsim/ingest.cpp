// ingest.cpp — TEST INFRASTRUCTURE: runs the action ingest's device code (csrc/ingest.cuh,
// ingest_actions_body<KIN>) on the CPU (g++, shim/cuda_runtime.h), one (env, agent) index after the
// other, in the order of the launch's thread indices.  Not product code.
#include "ingest.cuh"

using namespace vmas;

extern "C" {

// `agents`: n VmasAgentActions (host pointers); the state rows as in VmasState.  Returns 0, or -1 for n out of range.
int hostsim_ingest(int kin, const VmasAgentActions* agents, int n, int batch_dim, int n_entities, int n_agents_total,
                   float* pos, float* vel, float* rot, float* ang_vel, float* force, float* torque, int clamp,
                   uint8_t* bad_flag, float* steps) {
  if (n <= 0 || n > VMAS_MAX_INGEST_AGENTS) return -1;
  IngestArgs a;
  for (int i = 0; i < n; ++i) a.ag[i] = agents[i];
  a.st.pos = pos; a.st.vel = vel; a.st.rot = rot; a.st.ang_vel = ang_vel; a.st.force = force; a.st.torque = torque;
  a.bad_flag = bad_flag;
  a.steps = steps;
  a.n_entities = n_entities;
  a.n_agents_total = n_agents_total;
  a.n = n;
  a.batch_dim = batch_dim;
  a.clamp = clamp;
  const long total = (long)batch_dim * n;
  for (long idx = 0; idx < total; ++idx) {
    if (kin) ingest_actions_body<true>(a, idx);
    else ingest_actions_body<false>(a, idx);
  }
  return 0;
}

}  // extern "C"
