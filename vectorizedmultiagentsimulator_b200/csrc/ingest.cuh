// ingest.cuh — device part of the action ingest: decodes the policy's actions into agent.action.u and the
// force / torque rows (continuous, discrete and multi-discrete spaces; holonomic, forward, rotation and the
// kinematic models).  Included by vmas_b200.cu (the ingest kernels) and spec_kernel.cuh (the prologue of the
// one-kernel step); tests/hostsim compiles it with g++ and runs it on the CPU.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "geometry.cuh"
#include "vmas_b200.h"

namespace vmas {

// ---------------------------------------------------------------------------------------------
// action ingestion (ref environment.py:616-655, 707; dynamics/holonomic.py:14-15)
// ---------------------------------------------------------------------------------------------
struct IngestArgs {
  VmasAgentActions ag[VMAS_MAX_INGEST_AGENTS];
  VmasState st;
  uint8_t* bad_flag;
  float* steps;        // [B] step counter of the environment, or null
  int n_entities;      // E: row stride of pos / vel / rot / ang_vel
  int n_agents_total;  // A: row stride of force / torque
  int n;               // agents in this launch
  int batch_dim;
  int clamp;
};

// One continuous action component (ref environment.py:621, 633-655): NaN is flagged before the clamp and
// passes through it (torch.clamp keeps NaN; fmaxf(NaN, -r) would return -r), +-inf clamps to +-r, the range is
// checked after the clamp, and the scaling rounds once.  `bad` collects the flag.
DEVI float ingest_continuous(float v, const float r, const float m, const bool clamp, bool& bad) {
  const bool nan = v != v;
  if (clamp && !nan) v = fminf(fmaxf(v, -r), r);
  bad |= nan || (fabsf(v) > r);
  return v * m;
}

// One discrete action component (ref environment.py:656-706): index k of n choices becomes one of n evenly
// spaced values in [-r, r], scaled by m.  For odd n index 0 means "no force" and indices 1 .. n/2 shift down by
// one.  An index outside [0, n) sets `bad` and still decodes by the same formula.  (index, r and m by reference:
// then nvcc compiles ingest_actions_body to the same instructions as with this code written in line there.)
DEVI float ingest_discrete(const long long& index, const long long n, const float& r, const float& m, bool& bad) {
  long long k = index;
  bad |= k < 0 || k >= n;
  if (n % 2 != 0) {
    if (k == 0) k = n / 2;
    else if (k <= n / 2) k = k - 1;
  }
  const float v = ((float)k / (float)(n - 1)) * (2.f * r) - r;
  return v * m;
}

// ---- the kinematic action models (ref dynamics/diff_drive.py, kinematic_bicycle.py, drone.py) ---------
// Each integrates a small ODE over dt — classic RK4 or Euler, the reference's order of operations — to
// get the pose change the command asks for.
struct Pose3 {
  float x, y, yaw;
};
DEVI Pose3 diff_drive_f(float heading, float v, float w) {
  float s, c;
  sincosf(heading, &s, &c);
  Pose3 d = {v * c, v * s, w};
  return d;
}
DEVI Pose3 bicycle_f(float yaw, float steering, float v, float l_f, float l_r) {
  const float wheelbase = l_f + l_r;
  const float slip = atan2f(tanf(steering) * l_r / wheelbase, 1.f);
  float s, c;
  sincosf(yaw + slip, &s, &c);
  Pose3 d = {v * c, v * s, v / wheelbase * cosf(slip) * tanf(steering)};
  return d;
}
template <class F>
DEVI Pose3 integrate_pose(float yaw, float dt, bool rk4, F f) {
  const Pose3 k1 = f(yaw);
  if (!rk4) {
    Pose3 e = {dt * k1.x, dt * k1.y, dt * k1.yaw};
    return e;
  }
  const Pose3 k2 = f(yaw + dt * k1.yaw / 2.f);
  const Pose3 k3 = f(yaw + dt * k2.yaw / 2.f);
  const Pose3 k4 = f(yaw + dt * k3.yaw);
  const float w = dt / 6.f;
  Pose3 d = {w * (k1.x + 2.f * k2.x + 2.f * k3.x + k4.x), w * (k1.y + 2.f * k2.y + 2.f * k3.y + k4.y),
             w * (k1.yaw + 2.f * k2.yaw + 2.f * k3.yaw + k4.yaw)};
  return d;
}

struct Drone12 {
  float v[12];
};
DEVI Drone12 drone_f(const Drone12& s, float thrust, float tx, float ty, float tz, float mass, float Ixx, float Iyy,
                     float Izz, float g) {
  float sr, cr, sp, cp, sy, cy;
  sincosf(s.v[0], &sr, &cr);
  sincosf(s.v[1], &sp, &cp);
  sincosf(s.v[2], &sy, &cy);
  const float p = s.v[3], q = s.v[4], r = s.v[5];
  Drone12 d;
  d.v[0] = p;
  d.v[1] = q;
  d.v[2] = r;
  d.v[3] = (tx - (Iyy - Izz) * q * r) / Ixx;
  d.v[4] = (ty - (Izz - Ixx) * p * r) / Iyy;
  d.v[5] = (tz - (Ixx - Iyy) * p * q) / Izz;
  d.v[6] = (cr * sp * cy + sr * sy) * thrust / mass;
  d.v[7] = (cr * sp * sy - sr * cy) * thrust / mass;
  d.v[8] = (cr * cp) * thrust / mass - g;
  d.v[9] = s.v[6];
  d.v[10] = s.v[7];
  d.v[11] = s.v[8];
  return d;
}

// ---- the action models: force / torque from the decoded action u (ref dynamics/*.py) ---------------------------
// ingest_actions_body and the prologue of the one-kernel step (spec_kernel.cuh, spec_act_agent) both call these.
// (The drone's 12-state RK4 stays in ingest_actions_body: the prologue leaves drones to the ingest launch, and
// bicycles too: codegen.PROLOGUE_MODELS.)
// What each model writes into the slab: the agent's force row, its torque row
__host__ __device__ constexpr bool dyn_writes_force(int dyn) {
  return dyn == VMAS_DYN_HOLONOMIC || dyn == VMAS_DYN_HOLONOMIC_ROT || dyn == VMAS_DYN_FORWARD || dyn >= VMAS_DYN_DIFF_DRIVE;
}
__host__ __device__ constexpr bool dyn_writes_torque(int dyn) {
  return dyn == VMAS_DYN_HOLONOMIC_ROT || dyn == VMAS_DYN_ROTATION || dyn >= VMAS_DYN_DIFF_DRIVE;
}

// Forward: (u0, 0) rotated by the heading (ref dynamics/forward.py)
DEVI float2 forward_force(const float u0, const float rot) {
  float s, c;
  sincosf(rot, &s, &c);
  return make_float2(u0 * c - 0.f * s, u0 * s + 0.f * c);
}

// DiffDrive: the pose change of (v, w) = (u0, u1) over dt
DEVI Pose3 diff_drive_pose(const float v, const float w, const float yaw, const float dt, const bool rk4) {
  return integrate_pose(yaw, dt, rk4, [&](float h) { return diff_drive_f(h, v, w); });
}

// KinematicBicycle: the pose change of (v, steering) = (u0, u1) over dt, the steering clamped to +-lim
DEVI Pose3 bicycle_pose(const float v, const float steering, const float yaw, const float dt, const bool rk4,
                        const float l_f, const float l_r, const float lim) {
  const float steer = fminf(fmaxf(steering, -lim), lim);
  return integrate_pose(yaw, dt, rk4, [&](float h) { return bicycle_f(h, steer, v, l_f, l_r); });
}

// the force / torque that realise a kinematic model's pose change under the world's integrator (dynamics/common)
DEVI float2 kinematic_force(const Pose3& d, const float dt, const float mass, const float inertia, const float2 vel,
                            const float w0, float& torque) {
  const float dt2 = dt * dt;
  const float2 f = make_float2(mass * ((d.x - vel.x * dt) / dt2), mass * ((d.y - vel.y * dt) / dt2));
  torque = inertia * ((d.yaw - w0 * dt) / dt2);
  return f;
}

// KIN: the launch has an agent with a kinematic model (diff drive / bicycle / drone); the lean
// instantiation without that code needs half the registers, and most scenarios use it
template <bool KIN>
DEVI void ingest_actions_body(const IngestArgs& a, const long idx) {
  if (idx >= (long)a.batch_dim * a.n) return;
  const long env = idx / a.n;
  const int k = (int)(idx % a.n);
  const VmasAgentActions& ag = a.ag[k];
  const int sz = ag.action_size;
  float u[VMAS_MAX_ACTION_SIZE];
  bool bad = false;
  if (ag.action_kind == VMAS_ACT_CONTINUOUS) {
#pragma unroll
    for (int j = 0; j < VMAS_MAX_ACTION_SIZE; ++j) {
      u[j] = 0.f;
      if (j < sz) {
        u[j] = ingest_continuous(ag.actions[env * sz + j], ag.u_range[j], ag.u_multiplier[j], a.clamp, bad);
      }
    }
  } else {  // discrete / multi-discrete indices (ref environment.py:656-706)
    const long long* idx_in = reinterpret_cast<const long long*>(ag.actions);
    long long flat = ag.action_kind == VMAS_ACT_DISCRETE ? idx_in[env] : 0;
#pragma unroll
    for (int j = 0; j < VMAS_MAX_ACTION_SIZE; ++j) {
      u[j] = 0.f;
      if (j < sz) {
        const long long n = ag.nvec[j];
        long long k;
        if (ag.action_kind == VMAS_ACT_DISCRETE) {  // unravel the flat index of the cartesian product
          long long stride = 1;
          for (int m = j + 1; m < sz; ++m) stride *= ag.nvec[m];
          k = flat / stride;
          flat = flat % stride;
        } else {
          k = idx_in[env * sz + j];
        }
        u[j] = ingest_discrete(k, n, ag.u_range[j], ag.u_multiplier[j], bad);
      }
    }
  }
  if (bad && a.bad_flag) *a.bad_flag = 1;
  if (a.steps && k == 0) a.steps[env] = a.steps[env] + 1.f;
  const int dyn = ag.dynamics;
  const size_t row = (size_t)env * a.n_agents_total + ag.agent_index;
  const size_t ent = (size_t)env * a.n_entities + ag.entity_index;
  float2 force = make_float2(0.f, 0.f);
  float torque = 0.f;
  bool write_force = false, write_torque = false;
  if (dyn == VMAS_DYN_HOLONOMIC || dyn == VMAS_DYN_HOLONOMIC_ROT) {
    force = make_float2(u[0], u[1]);
    write_force = true;
    if (dyn == VMAS_DYN_HOLONOMIC_ROT) {
      torque = u[2];
      write_torque = true;
    }
  } else if (dyn == VMAS_DYN_FORWARD) {
    force = forward_force(u[0], a.st.rot[ent]);
    write_force = true;
  } else if (dyn == VMAS_DYN_ROTATION) {
    torque = u[0];
    write_torque = true;
  } else if (KIN && dyn >= VMAS_DYN_DIFF_DRIVE) {
    const float dt = ag.dyn_params[0], mass = ag.dyn_params[1], inertia = ag.dyn_params[2];
    const bool rk4 = ag.dyn_params[3] != 0.f;
    const float yaw = a.st.rot[ent];
    Pose3 d;
    if (dyn == VMAS_DYN_DIFF_DRIVE) {
      d = diff_drive_pose(u[0], u[1], yaw, dt, rk4);
    } else if (dyn == VMAS_DYN_BICYCLE) {
      d = bicycle_pose(u[0], u[1], yaw, dt, rk4, ag.dyn_params[4], ag.dyn_params[5], ag.dyn_params[6]);
    } else {  // drone: thrust gets the hover feed-forward (in place on the action, as the reference does)
      const float Ixx = ag.dyn_params[4], Iyy = ag.dyn_params[5], Izz = ag.dyn_params[6], g = ag.dyn_params[7];
      u[0] = u[0] + mass * g;
      const float thrust = u[0], tx = u[1], ty = u[2], tz = u[3];
      float* ds = ag.dyn_state + (size_t)env * 12;
      Drone12 s;
#pragma unroll
      for (int j = 0; j < 12; ++j) s.v[j] = ds[j];
      const float2 p = reinterpret_cast<const float2*>(a.st.pos)[ent];
      s.v[9] = p.x;
      s.v[10] = p.y;
      s.v[2] = yaw;
      auto f = [&](const Drone12& x) { return drone_f(x, thrust, tx, ty, tz, mass, Ixx, Iyy, Izz, g); };
      auto axpy = [&](const Drone12& x, float h, const Drone12& kk) {
        Drone12 o;
#pragma unroll
        for (int j = 0; j < 12; ++j) o.v[j] = x.v[j] + h * kk.v[j] / 2.f;
        return o;
      };
      Drone12 delta;
      const Drone12 k1 = f(s);
      if (!rk4) {
#pragma unroll
        for (int j = 0; j < 12; ++j) delta.v[j] = dt * k1.v[j];
      } else {
        const Drone12 k2 = f(axpy(s, dt, k1));
        const Drone12 k3 = f(axpy(s, dt, k2));
        Drone12 s4;
#pragma unroll
        for (int j = 0; j < 12; ++j) s4.v[j] = s.v[j] + dt * k3.v[j];
        const Drone12 k4 = f(s4);
#pragma unroll
        for (int j = 0; j < 12; ++j) delta.v[j] = (dt / 6.f) * (k1.v[j] + 2.f * k2.v[j] + 2.f * k3.v[j] + k4.v[j]);
      }
#pragma unroll
      for (int j = 0; j < 12; ++j) ds[j] = s.v[j] + delta.v[j];
      d.x = delta.v[6];
      d.y = delta.v[7];
      d.yaw = delta.v[5];
    }
    force = kinematic_force(d, dt, mass, inertia, reinterpret_cast<const float2*>(a.st.vel)[ent], a.st.ang_vel[ent], torque);
    write_force = write_torque = true;
  }
#pragma unroll
  for (int j = 0; j < VMAS_MAX_ACTION_SIZE; ++j)
    if (j < sz) ag.u[env * sz + j] = u[j];
  if (write_force) reinterpret_cast<float2*>(a.st.force)[row] = force;
  if (write_torque) a.st.torque[row] = torque;
}

}  // namespace vmas
