/*
 * vmas_b200.h — C ABI of the H100 (sm_90a) physics hot path of VMAS.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  Every entry point
 * replaces one piece of the reference's pure-Python/PyTorch hot path
 * (vmas/simulator/core.py); the Python host (ctypes, see
 * vectorizedmultiagentsimulator_b200/_native.py and INTEGRATION.md) passes device pointers of
 * tensors it owns plus the CUDA stream to launch on.  Nothing here allocates device memory or
 * synchronises the device.
 *
 * State layout (all fp32, contiguous, one CUDA device):
 *   pos     [B, E, 2]   vel     [B, E, 2]   rot   [B, E]   ang_vel [B, E]
 *   force   [B, A, 2]   torque  [B, A]      (A = agents; E follows world.entities order)
 *
 * Return convention: >= 0 on success (for launch functions: the number of kernels launched),
 * < 0 on error; vmas_b200_last_error() then returns a message for the calling thread.
 */
#ifndef VMAS_B200_H
#define VMAS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VMAS_B200_ABI_VERSION 2

/* shape kinds (ent_i32[:,0]) */
enum { VMAS_SHAPE_SPHERE = 0, VMAS_SHAPE_BOX = 1, VMAS_SHAPE_LINE = 2 };
/* work-item kinds (item_i32[:,0]), in force-accumulation order (ref core.py:2175-2189) */
enum { VMAS_K_JOINT = 0, VMAS_K_SS = 1, VMAS_K_LS = 2, VMAS_K_LL = 3, VMAS_K_BS = 4, VMAS_K_BL = 5, VMAS_K_BB = 6 };

/* entity flag bits (ent_i32[:,1]) */
enum {
  VMAS_F_MOVABLE = 1 << 0, VMAS_F_ROTATABLE = 1 << 1, VMAS_F_HOLLOW = 1 << 2, VMAS_F_AGENT = 1 << 3,
  VMAS_F_LIN_FRIC = 1 << 4, VMAS_F_ANG_FRIC = 1 << 5, VMAS_F_GRAVITY = 1 << 6, VMAS_F_MAX_SPEED = 1 << 7,
  VMAS_F_V_RANGE = 1 << 8, VMAS_F_MAX_F = 1 << 9, VMAS_F_F_RANGE = 1 << 10, VMAS_F_MAX_T = 1 << 11,
  VMAS_F_T_RANGE = 1 << 12, VMAS_F_TRIG = 1 << 13, VMAS_F_GRAVITY_ENV = 1 << 14,
  /* per-env mass / friction coefficients, read from the ent_params table of vmas_b200_world_step_params */
  VMAS_F_MASS_ENV = 1 << 15, VMAS_F_LIN_FRIC_ENV = 1 << 16, VMAS_F_ANG_FRIC_ENV = 1 << 17
};
/* columns of ent_f32 [E, 20] */
enum {
  VMAS_EF_D0 = 0, VMAS_EF_D1, VMAS_EF_MASS, VMAS_EF_INERTIA, VMAS_EF_DRAG_MULT, VMAS_EF_LIN_FRIC,
  VMAS_EF_ANG_FRIC, VMAS_EF_GRAV_X, VMAS_EF_GRAV_Y, VMAS_EF_MAX_SPEED, VMAS_EF_V_RANGE, VMAS_EF_MAX_F,
  VMAS_EF_F_RANGE, VMAS_EF_MAX_T, VMAS_EF_T_RANGE, VMAS_EF_CIRC_R, VMAS_EF_R_PLUS_LMD,
  /* VMAS_F_MASS_ENV: moment of inertia = fp32(fp32(K0 * mass) * K1) (ref core.py:123-124, 160-161, 187-188) */
  VMAS_EF_INERTIA_K0, VMAS_EF_INERTIA_K1,
  VMAS_EF_COLS = 20
};
/* columns of the per-env parameter table ent_params [B, E, VMAS_EP_COLS] */
enum { VMAS_EP_MASS = 0, VMAS_EP_LIN_FRIC = 1, VMAS_EP_ANG_FRIC = 2, VMAS_EP_COLS = 4 };
/* columns of item_f32 [NI, 8] */
enum {
  VMAS_IF_BROAD_THR = 0, VMAS_IF_DMIN_BASE, VMAS_IF_AX, VMAS_IF_AY, VMAS_IF_BX, VMAS_IF_BY, VMAS_IF_DIST,
  VMAS_IF_FIXED_ROT, VMAS_IF_COLS
};
/* item flag bits (item_i32[:,3] low byte); bits 8.. hold (mask bit index + 1), 0 = never masked */
enum { VMAS_IFLAG_JOINT_ROTATE = 1, VMAS_IFLAG_JOINT_ROT_PER_ENV = 2, VMAS_IFLAG_ALWAYS_ACTIVE = 4 };

/* World scalars (ref World.__init__, core.py:1091-1150).  Host memory, passed by pointer. */
typedef struct VmasWorldConfig {
  int32_t batch_dim;      /* B */
  int32_t n_entities;     /* E */
  int32_t n_agents;       /* A */
  int32_t n_items;        /* joints + candidate collision pairs */
  int32_t n_joints;       /* items [0, n_joints) are joint constraints */
  int32_t n_masked;       /* items that obey the batch-wide broad-phase mask (line/box pairs) */
  int32_t substeps;       /* S */
  int32_t has_x_semidim, has_y_semidim, has_world_gravity;
  float sub_dt;           /* fp32(dt / S) */
  float x_semidim, y_semidim;
  float collision_force, joint_force, torque_constraint_force, contact_margin;
  float gravity_x, gravity_y;
} VmasWorldConfig;

/* Plan tables compiled on the host from the world's static structure.  DEVICE pointers. */
typedef struct VmasPlanTables {
  const float*   ent_f32;     /* [E, VMAS_EF_COLS] */
  const int32_t* ent_i32;     /* [E, 4]: shape, flags, agent index, - */
  const float*   item_f32;    /* [NI, VMAS_IF_COLS] */
  const int32_t* item_i32;    /* [NI, 4]: kind, a, b, flags | (mask bit + 1) << 8 */
  const int32_t* inc_off;     /* [E + 1] CSR offsets: items incident to each entity */
  const int32_t* inc;         /* item * 2 + side, ascending item order */
  const int32_t* sched;       /* [n_rounds, group] item per lane, -1 = idle; rounds are kind-uniform
                                 (lane-per-entity mapping only; ignored when group == 1) */
  const int32_t* masked_items;/* [n_masked] item index of each mask bit */
  const float*   joint_rot;   /* [B, n_joints] per-env fixed rotations, or NULL */
  const float*   ent_gravity; /* [B, E, 2] per-env gravity of entities flagged VMAS_F_GRAVITY_ENV, or NULL
                                 (ref core.py:594-601, 2049-2052: Entity.gravity given as a tensor) */
  int32_t n_rounds;
  int32_t group;              /* lanes per env: 1 = one thread per env (default), or 8, 16, 32; with a
                                 specialization: 1, or VMAS_GROUP_TILE = the warp-tile kernel (a warp owns
                                 32 envs; far tests per env, then the narrow phase of the near (item, env)
                                 pairs compacted over the warp's lanes; see csrc/spec_tile_kernel.cuh);
                                 without one: VMAS_GROUP_BLOCK = a thread block per env (step_block_kernel) */
  int32_t ents_per_lane;      /* 1, 2 or 4 (E <= group * ents_per_lane) */
  int32_t specialization;     /* index from vmas_b200_find_specialization(), or -1: generic kernels */
  /* env scheduling of the specialised thread-per-env kernel (both optional, may be NULL): */
  const int32_t* env_order;   /* [B] permutation: thread t steps env env_order[t] (vmas_b200_build_env_order) */
  uint32_t* env_signature;    /* [B] out: bit (i & 31) set iff work item i produced a force in this step */
} VmasPlanTables;

#define VMAS_GROUP_TILE (-8)
/* A thread block per env, its state in shared memory as [field][entity]: for worlds of up to
 * VMAS_BLOCK_MAX_ENTITIES entities whose one-thread-per-env layout does not fit in shared memory. */
#define VMAS_GROUP_BLOCK (-16)
#define VMAS_BLOCK_MAX_ENTITIES 1024

/* The state slab.  DEVICE pointers. */
typedef struct VmasState {
  float* pos; float* vel; float* rot; float* ang_vel; float* force; float* torque;
} VmasState;

/* One (source, destination, size) piece of vmas_b200_copy_buffers().  DEVICE pointers. */
typedef struct VmasCopySegment {
  const void* src;
  void* dst;
  size_t bytes;
} VmasCopySegment;
#define VMAS_MAX_COPY_SEGMENTS 64

int vmas_b200_abi_version(void);
const char* vmas_b200_last_error(void);

/*
 * World-specialised kernels.  The library carries ahead-of-time specialisations of the substep
 * kernel for a set of worlds (csrc/generated/, see codegen.py), keyed by a 64-bit hash of the
 * world description.  find returns an index for VmasPlanTables.specialization, or -1.
 */
int vmas_b200_num_specializations(void);
int vmas_b200_find_specialization(uint64_t world_hash);
const char* vmas_b200_specialization_name(int index);
/*
 * Run-time specialisation.  Any world can get the specialised kernels: the host generates the
 * world's constexpr tables (codegen.emit_world), compiles csrc/spec_kernel.cuh for them into a small
 * shared object (simulator/jit.py: nvcc for sm_90a, cached by world hash) and registers the object's
 * launch functions here.  `launch` / `launch_tile`: addresses of
 *     cudaError_t fn(const vmas::SpecArgs&, cudaStream_t)      (launch_tile may be NULL)
 * `spec_args_bytes` = sizeof(vmas::SpecArgs) as the object was compiled (layout check).
 * Returns the index for VmasPlanTables.specialization (the existing one if the hash is known).
 */
#define VMAS_MAX_RUNTIME_SPECS 256
int vmas_b200_register_specialization(uint64_t world_hash, int32_t n_entities, int32_t n_items, void* launch,
                                      void* launch_tile, int32_t spec_args_bytes);
/* 1 if the specialization also has the warp-tile kernel (VmasPlanTables.group = VMAS_GROUP_TILE) */
int vmas_b200_specialization_has_tile(int index);

/*
 * One World.step(): S substeps of force accumulation -> contact/joint resolution ->
 * semi-implicit Euler, in place on `st`.  Replaces ref core.py:1972-2015 (and everything it
 * calls: :2018-2908, physics.py, joints.py:186-216).
 *   mask        device scratch, uint32[(n_masked + 31) / 32 + 1], zero before the first call; only
 *               used when the world has line/box pairs and exact_broad_phase != 0
 *               (batch-wide pair activation, ref core.py:2797-2801).
 * Sphere-only worlds run all S substeps in ONE launch; otherwise 2 launches per substep.
 */
int vmas_b200_world_step(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                         uint32_t* mask, int exact_broad_phase, void* cuda_stream);

/*
 * vmas_b200_world_step for a world whose entities carry per-env physical parameters (domain
 * randomisation: ref core.py:2043-2102, 2870 with a [B, 1] Entity.mass / friction coefficient).
 *   ent_params  device fp32 [B, E, VMAS_EP_COLS]: mass, linear-friction coefficient, angular-friction
 *               coefficient, unused.  Only the columns an entity's VMAS_F_*_ENV flags name are read, and only
 *               for flagged entities; the rest of the table is never touched.  NULL: no entity is flagged
 *               (vmas_b200_world_step is this call with NULL).  A specialised world with flagged entities
 *               called with NULL fails with an error; the generic kernels then read the description's
 *               placeholder scalars, never the table.
 * Per-env gravity (VMAS_F_GRAVITY_ENV) is read from VmasPlanTables.ent_gravity as before.
 */
int vmas_b200_world_step_params(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const float* ent_params,
                                const VmasState* st, uint32_t* mask, int exact_broad_phase, void* cuda_stream);

/*
 * Same as vmas_b200_world_step, additionally recording two caller-owned CUDA events
 * (cudaEvent_t, may be NULL) on the stream: `ev_begin` right before the first substep kernel
 * and `ev_end` right after the last one.  The broad-phase launches of worlds with line/box
 * pairs fall inside the bracket only when S > 1.  Used by bench.py for the roofline figure.
 */
int vmas_b200_world_step_timed(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                               uint32_t* mask, int exact_broad_phase, void* cuda_stream,
                               void* ev_begin, void* ev_end);

/* Same, for a sub-range of substeps [first_substep, first_substep + n_substeps) (testing). */
int vmas_b200_world_substeps(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                             uint32_t* mask, int exact_broad_phase, int first_substep, int n_substeps,
                             void* cuda_stream);

/*
 * World.cast_rays() (ref core.py:1662-1786) for one source entity.
 *   targets      device int32[n_targets]: entity indices the rays may hit
 *   angles       device fp32 [B, n_rays]
 *   add_rot_of   >= 0: add rot[:, add_rot_of] to every angle (Lidar.measure, ref sensors.py:116-121)
 *   out          device fp32 [B, n_rays]
 */
int vmas_b200_cast_rays(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                        int32_t src_entity, const int32_t* targets, int32_t n_targets,
                        const float* angles, int32_t n_rays, int32_t add_rot_of, float max_range,
                        float* out, void* cuda_stream);

/*
 * Batched LIDAR: every ray of `n_sensors` sensors in ONE launch (the reference runs one
 * World.cast_rays per agent per step, sensors.py:116-121).  All sensors share `n_rays`.
 *   src          device int32[Q]      source entity of each sensor (its rotation is added to the angles)
 *   target_off   device int32[Q + 1]  CSR offsets into `targets`
 *   targets      device int32[...]    entity indices each sensor's rays may hit
 *   angles       device fp32 [Q, n_rays]  sensor-frame ray angles
 *   max_range    device fp32 [Q]
 *   out          device fp32; sensor q's reading of (env, ray) goes to
 *                out[out_offsets[q] + env * out_env_stride + ray]
 *   out_offsets  device int64[Q] or NULL (= q * B * n_rays: a dense [Q, B, n_rays] block)
 *   out_env_stride  elements between consecutive envs (0 = n_rays).  A stride > n_rays lets the
 *                readings land directly in columns of an observation block [A, B, F].
 *   flags        VMAS_RAYS_RANGE_MINUS_DISTANCE: store max_range - distance (the form
 *                scenarios/navigation.py:260 feeds to the policy) instead of the distance
 */
#define VMAS_RAYS_RANGE_MINUS_DISTANCE 1
/* the caller guarantees every entity in `targets` is a sphere: a kernel without box / line code */
#define VMAS_RAYS_SPHERE_TARGETS 2
int vmas_b200_cast_rays_batched(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                int32_t n_sensors, const int32_t* src, const int32_t* target_off,
                                const int32_t* targets, const float* angles, const float* max_range,
                                int32_t n_rays, float* out, const int64_t* out_offsets, int64_t out_env_stride,
                                int32_t flags, void* cuda_stream);

/*
 * Observation assembly: fills the slab-derived columns of an observation block out[R, B, F] in one
 * launch (the reference builds each agent's observation with per-term slices and torch.cat,
 * e.g. scenarios/balance.py:236-262, navigation.py:252-265).
 *   columns  device int32[R * F * 4]: per (row, column) {op, source a, source b, param}
 *            op: VMAS_OBS_SKIP (left untouched: LIDAR readings, scenario-specific terms),
 *                VMAS_OBS_COPY a, VMAS_OBS_DIFF a - b, VMAS_OBS_REMAINDER torch.remainder(a, param)
 *            source: (field << 24) | element offset within the env's row of that field
 *                    (pos / vel: 2 * entity + axis; rot / ang_vel: entity)
 *            param: fp32 bit pattern
 */
#define VMAS_OBS_SKIP 0
#define VMAS_OBS_COPY 1
#define VMAS_OBS_DIFF 2
#define VMAS_OBS_REMAINDER 3
/* a per-env fp32 value another producer holds (a flag the scenario's step program stored, say):
 * source a = index into `buffers` (vmas_b200_gather_observations_buffers); the launch that wrote the buffer
 * must precede this one in stream order */
#define VMAS_OBS_BUFFER 4
/* (whole-step kernels only: the column is register `source a` of the step program that ran in the same thread) */
#define VMAS_OBS_REG 5
#define VMAS_OBS_MAX_BUFFERS 8
#define VMAS_OBS_POS 0
#define VMAS_OBS_VEL 1
#define VMAS_OBS_ROT 2
#define VMAS_OBS_ANG_VEL 3
int vmas_b200_gather_observations(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* columns,
                                  int32_t n_rows, int32_t width, float* out, void* cuda_stream);
/* The same with VMAS_OBS_BUFFER columns: `buffers` = n_buffers device pointers to fp32 [B] arrays. */
int vmas_b200_gather_observations_buffers(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* columns,
                                          int32_t n_rows, int32_t width, float* out, const float* const* buffers,
                                          int32_t n_buffers, void* cuda_stream);

/*
 * Post-step program: the scenario's reward / done glue (distance and overlap queries, the distance-shaping
 * pattern, elementwise operations on per-env scalars) as a short instruction list interpreted by one
 * thread per env, launched TOGETHER with the observation gather (the blocks with blockIdx.y == n_rows run
 * the program).  Replaces the chain of small torch kernels a scenario's reward() / done() issue every step
 * (ref scenarios/balance.py:197-263).  Registers hold fp32 values, booleans are 0 / 1.
 *   op               operands
 *   OVERLAP / DISTANCE / CENTER_DISTANCE   dst <- query(entity arg & 0xFFFF, entity arg >> 16)
 *   SHAPING          dst <- buffers[a][env] - d * imm;  dst + 1 <- d = |pos_a - pos_b|;  buffers[a][env] <- d * imm
 *   LOAD_F32 / LOAD_BOOL   dst <- buffers[a][env]          CONST   dst <- imm
 *   ADD SUB MUL MIN MAX OR AND LT LE   dst <- a op b       NEG NOT   dst <- op a
 *   WHERE            dst <- a != 0 ? b : register (arg & 0xFF)
 *   STORE_F32 / STORE_BOOL   buffers[b][env] <- a
 *   STEP_COUNT       dst <- the env's step counter after this step's increment; `a`: the buffer slot of the counter
 *                    (Environment.steps).  A load of buffers[a][env] everywhere but in step_env_kernel, which counts
 *                    the step in its prologue and hands the sum over in a register.
 * `columns`, `n_rows`, `width`, `obs_out`: as vmas_b200_gather_observations (or NULL / 0: program only).
 */
#define VMAS_PROG_MAX_INSTR 64
#define VMAS_PROG_MAX_BUFFERS 32
#define VMAS_PROG_REGS 32
enum {
  VMAS_OP_OVERLAP = 1, VMAS_OP_DISTANCE, VMAS_OP_CENTER_DISTANCE, VMAS_OP_SHAPING, VMAS_OP_LOAD_F32, VMAS_OP_LOAD_BOOL,
  VMAS_OP_CONST, VMAS_OP_ADD, VMAS_OP_SUB, VMAS_OP_MUL, VMAS_OP_MIN, VMAS_OP_MAX, VMAS_OP_NEG, VMAS_OP_OR, VMAS_OP_AND,
  VMAS_OP_NOT, VMAS_OP_LT, VMAS_OP_LE, VMAS_OP_WHERE, VMAS_OP_STORE_F32, VMAS_OP_STORE_BOOL, VMAS_OP_STEP_COUNT
};
typedef struct VmasProgInstr {
  uint8_t op, dst, a, b;
  int32_t arg;
  float imm;
} VmasProgInstr;
typedef struct VmasStepProgram {
  int32_t n_instr;
  int32_t reserved;
  VmasProgInstr instr[VMAS_PROG_MAX_INSTR];
  void* buffers[VMAS_PROG_MAX_BUFFERS];  /* device pointers: per-env fp32 or uint8 arrays [B] */
} VmasStepProgram;
int vmas_b200_post_step(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                        const VmasStepProgram* program, const int32_t* columns, int32_t n_rows, int32_t width,
                        float* obs_out, void* cuda_stream);

/*
 * Distance shaping for K entity pairs in one launch — the reward pattern of
 * scenarios/balance.py:197-214, navigation.py:203-216, transport.py:139-152:
 *     dist = |pos_a - pos_b|;  rew = prev - dist * factor;  prev <- dist * factor   (fp32, in this order)
 *   pairs  device int32[K, 2];  prev device fp32[K, B] (in / out);  dist fp32[K, B] or NULL;  rew fp32[K, B]
 */
int vmas_b200_distance_shaping(const VmasWorldConfig* cfg, const VmasState* st, const int32_t* pairs,
                               int32_t n_pairs, float factor, float* prev, float* dist, float* rew,
                               void* cuda_stream);

/*
 * Env scheduling.  Envs are independent, so WHICH thread steps an env is free; the thread-per-env
 * kernel diverges when the 32 envs of a warp need different narrow-phase work (different contacts).
 * Contacts persist over steps, so grouping envs by the signature the previous step recorded
 * (VmasPlanTables.env_signature) makes a warp's envs take the same branches.  This builds the
 * permutation: the envs of every chunk of `chunk` (256, 512, 1024 or 2048) consecutive envs sorted by
 * (signature, env index) — chunk-local so that a warp's rows stay within a small window of each state
 * array (a global sort makes the kernel memory-bound).  Results never depend on the order.
 *   signature  device uint32[B];  order  device int32[B] (out)
 * One launch; meant to be called every few steps, not every step.
 */
int vmas_b200_build_env_order(const uint32_t* signature, int32_t batch_dim, int32_t* order, int32_t chunk,
                              void* cuda_stream);
/* cudaLimitMaxL2FetchGranularity of the current device (32 / 64 / 128 bytes); returns what the device reports. */
int vmas_b200_set_l2_fetch_granularity(int32_t bytes);

/*
 * Copies up to VMAS_MAX_COPY_SEGMENTS device buffers in ONE kernel launch (an SM copy, not a copy
 * engine: it does not queue behind a concurrent host download).  Used to hand out fresh copies of
 * the outputs a captured Environment.step writes into static buffers (the reference returns new
 * tensors from every step, ref environment/environment.py:254-309).
 */
int vmas_b200_copy_buffers(const VmasCopySegment* segs, int32_t n_segs, void* cuda_stream);
/*
 * The same, where segment i may convert: kinds[i] = VMAS_DTYPE_F32 copies `bytes` bytes as above;
 * VMAS_DTYPE_F16 / VMAS_DTYPE_BF16 read `bytes` bytes of fp32 values (a multiple of 4, `src` 4-byte aligned) and
 * write each rounded to nearest even to that 16-bit type (`bytes` / 2 bytes, `dst` 2-byte aligned): overflow goes
 * to +-inf, -0 stays -0, a NaN stays NaN.  16-bit observations of a captured Environment.step are handed out so.
 */
#define VMAS_DTYPE_F32 0
#define VMAS_DTYPE_F16 1
#define VMAS_DTYPE_BF16 2
int vmas_b200_copy_buffers_convert(const VmasCopySegment* segs, const int32_t* kinds, int32_t n_segs,
                                   void* cuda_stream);


/*
 * K entity pairs in one launch: mode 0 = World.get_distance (fp32), 1 = World.is_overlapping
 * (uint8), 2 = distance between the two centres (fp32; the quantity World.collides thresholds,
 * ref core.py:2797-2799).   pairs: device int32[K, 2];  out: [K, B].
 * `mode | VMAS_QUERY_SPHERES`: the caller guarantees every entity named in `pairs` is a sphere;
 * the launch then uses a kernel without the box / line closest-point code (same results).
 */
#define VMAS_QUERY_SPHERES 0x100
int vmas_b200_pair_query_batched(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                 const int32_t* pairs, int32_t n_pairs, int32_t mode, void* out,
                                 void* cuda_stream);

/*
 * World.get_distance (mode 0 -> fp32 out[B]) / World.is_overlapping (mode 1 -> uint8 out[B]) for
 * the entity pair (a, b).  Replaces ref core.py:1822-1969.
 */
int vmas_b200_pair_query(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                         int32_t a, int32_t b, int32_t mode, void* out, void* cuda_stream);

/* World.get_distance_from_point (ref core.py:1788-1820): point fp32 [B, 2] -> out fp32 [B]. */
int vmas_b200_point_query(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                          int32_t entity, const float* point, float* out, void* cuda_stream);

/*
 * Action ingestion for continuous actions: validates, scales and routes the policy's actions of up
 * to VMAS_MAX_INGEST_AGENTS agents in ONE launch.  Replaces, per agent, the chain of eager ops of
 * ref environment.py:616-655, 707 (`Environment._set_action`: nan / range asserts, optional clamp,
 * `u = action * u_multiplier`) and the Holonomic / HolonomicWithRotation dynamics
 * (ref dynamics/holonomic.py:14-15, holonomic_with_rot.py: `state.force = u[:, :2]`,
 * `state.torque = u[:, 2]`).
 *   actions      device fp32 [B, action_size], contiguous (discrete spaces: int64, see action_kind)
 *   u            device fp32 [B, action_size]: receives action * u_multiplier (agent.action.u)
 *   dynamics     which action -> force / torque model runs in the same launch (VMAS_DYN_*):
 *                  holonomic (force <- u[0:2]; ref dynamics/holonomic.py:14-15), with rotation (+ torque <- u[2];
 *                  holonomic_with_rot.py), forward (u[0] along the heading; forward.py), rotation (torque <- u[0];
 *                  roatation.py), differential drive (diff_drive.py:14-82), kinematic bicycle
 *                  (kinematic_bicycle.py:14-111), drone (drone.py:17-166) — the last three integrate their ODE
 *                  over dt (Euler or RK4) and back-solve the force / torque that realise the pose change under
 *                  the world's semi-implicit Euler step (dynamics/common + each model's process_action);
 *                  VMAS_DYN_NONE: only fill `u` (another model consumes it afterwards)
 *   entity_index entity row of the agent in pos / vel / rot (forward and the kinematic models read them)
 *   dyn_params   [0] dt  [1] mass  [2] moment of inertia  [3] 1 = RK4, 0 = Euler;
 *                bicycle: [4] l_f  [5] l_r  [6] max steering angle;  drone: [4] I_xx  [5] I_yy  [6] I_zz  [7] g
 *   dyn_state    drone only: device fp32 [B, 12] (roll pitch yaw | p q r | vx vy vz | x y z), updated in place
 *   bad_flag     device uint8[1] or NULL: set to 1 if any action is NaN (with or without `clamp`: a NaN passes
 *                the clamp unchanged) or outside +-u_range after the optional clamp (the reference asserts;
 *                here the host reads the flag back asynchronously)
 */
#define VMAS_MAX_INGEST_AGENTS 16
#define VMAS_MAX_ACTION_SIZE 8
enum {
  VMAS_DYN_NONE = -1, VMAS_DYN_HOLONOMIC = 0, VMAS_DYN_HOLONOMIC_ROT = 1, VMAS_DYN_FORWARD = 2, VMAS_DYN_ROTATION = 3,
  VMAS_DYN_DIFF_DRIVE = 4, VMAS_DYN_BICYCLE = 5, VMAS_DYN_DRONE = 6
};
typedef struct VmasAgentActions {
  const float* actions;
  float* u;
  int32_t action_size;
  int32_t agent_index;   /* row in force / torque */
  int32_t dynamics;
  int32_t entity_index;  /* row in pos / vel / rot / ang_vel */
  float u_range[VMAS_MAX_ACTION_SIZE];
  float u_multiplier[VMAS_MAX_ACTION_SIZE];
  float dyn_params[8];
  float* dyn_state;
  /* discrete action spaces (ref environment/environment.py:656-706): `actions` is then device int64 —
   * [B, 1] holding the flat index of the cartesian product of the components (VMAS_ACT_DISCRETE) or
   * [B, action_size] with one index per component (VMAS_ACT_MULTIDISCRETE); component j has nvec[j]
   * choices and decodes to  u_j = (k / (n - 1)) * (2 u_range_j) - u_range_j  with the reference's
   * re-ordering for odd n (index 0 = "no force").  An index outside [0, n) raises `bad_flag`. */
  int32_t action_kind;   /* VMAS_ACT_CONTINUOUS (0) | VMAS_ACT_DISCRETE | VMAS_ACT_MULTIDISCRETE */
  int32_t nvec[VMAS_MAX_ACTION_SIZE];
} VmasAgentActions;
enum { VMAS_ACT_CONTINUOUS = 0, VMAS_ACT_DISCRETE = 1, VMAS_ACT_MULTIDISCRETE = 2 };

/* `steps`: device fp32 [B] or NULL — the environment's per-env step counter (ref environment.py:396,
 * `self.steps += 1`), incremented here so that it does not cost a launch of its own. */
int vmas_b200_ingest_actions(const VmasWorldConfig* cfg, const VmasState* st, const VmasAgentActions* agents,
                             int32_t n_agents, int32_t clamp, uint8_t* bad_flag, float* steps, void* cuda_stream);

/*
 * PID velocity controller (ref vmas/simulator/controllers/velocity_controller.py:113-125, process_force):
 *     err = u - vel;  [accum += dt * err, clamped to +-windup;]  rate = Td * (err - prev) / dt;  prev <- err;
 *     u <- gain * (err [+ accum / Ti] + rate) * mass                          (fp32, in this order, in place)
 *   u      device fp32 [B, 2] (the agent's action, a velocity target on entry, a force on exit)
 *   accum, prev  device fp32 [B, 2] controller state;  inv_ti = 1 / Ti or 0 (no integrator);
 *   windup < 0: no anti-windup clamp
 */
int vmas_b200_velocity_controller(const VmasWorldConfig* cfg, const VmasState* st, int32_t entity, float* u,
                                  float* accum, float* prev, float gain, float inv_ti, float td, float dt,
                                  float windup, float mass, void* cuda_stream);

/* The same plus the broad phase of the step's FIRST substep (vmas_b200_broad_phase into `mask`) in one
 * launch; the following vmas_b200_world_step must then be told so (`exact_broad_phase` = 2).  Only valid
 * when nothing moves an entity between the two calls. */
int vmas_b200_ingest_actions_broad_phase(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                                         const VmasAgentActions* agents, int32_t n_agents, int32_t clamp,
                                         uint8_t* bad_flag, float* steps, uint32_t* mask, void* cuda_stream);

/*
 * One Environment.step() of a set-up environment in ONE call (replaces the host side of ref
 * environment/environment.py:254-309 once the step's work is known): in stream order
 *   1. vmas_b200_ingest_actions[_broad_phase] on the caller's action tensors (n_agents > 0);
 *   2. the step proper: either `graph_exec` (a cudaGraphExec_t holding the physics step and the scenario's
 *      callbacks, captured by the caller) is launched, or — `graph_exec` NULL — vmas_b200_world_step followed
 *      by vmas_b200_post_step (`program` / `columns` as there; both NULL: physics only) — or, with
 *      `fused_kernel`, ONE launch doing both;
 *   3. vmas_b200_copy_buffers (with `seg_kind`: vmas_b200_copy_buffers_convert) handing results out: segment i is
 *      copied to out_blocks[seg_block[i]] + (byte offset held in segs[i].dst), so that a caller allocating fresh
 *      result blocks every step only fills in `out_blocks` (n_segs may be 0: see `obs_block` / `mirror_*` below).
 * `ingest_mask` non-NULL: the ingest launch also builds the first substep's broad-phase mask (then
 * `exact_broad_phase` must be 2 in direct mode, and the captured graph must have been captured that way).
 * Returns the number of kernels this call launched itself (the graph's nodes are not counted).
 */
/*
 * Registers a WHOLE-STEP kernel compiled at run time for one (world, step program, observation plan): the
 * specialised substep kernel with the program and the observation rows as its epilogue (csrc/spec_kernel.cuh,
 * step_fused_kernel; built by vectorizedmultiagentsimulator_b200/jit.py).  `launch`:
 * cudaError_t (*)(const SpecArgs&, const EpiArgs&, cudaStream_t); `launch_env` (or NULL): the same kernel with
 * the action ingest and the broad phase as its prologue (step_env_kernel),
 * cudaError_t (*)(const SpecArgs&, const EpiArgs&, const ActArgs&, cudaStream_t).  Returns a handle > 0 for
 * VmasEnvStep.fused_kernel (the same key returns the same handle).
 */
int vmas_b200_register_step_kernel(uint64_t key, int32_t n_entities, int32_t n_items, void* launch, void* launch_env,
                                   int32_t spec_args_bytes, int32_t epi_args_bytes, int32_t act_args_bytes);

/* Number of nodes of a cudaGraph_t (a caller that captured a step checks whether the graph holds only
 * this library's launches: then VmasEnvStep's direct mode can stand in for it). */
int vmas_b200_graph_num_nodes(void* cuda_graph);

#define VMAS_MAX_OUT_BLOCKS 8
typedef struct VmasEnvStep {
  const VmasWorldConfig* cfg;
  const VmasPlanTables* tb;
  const VmasState* st;
  /* 1 */
  const VmasAgentActions* agents;
  int32_t n_agents, clamp;
  uint8_t* bad_flag;
  float* steps;
  uint32_t* ingest_mask;
  /* 2 */
  void* graph_exec;
  uint32_t* mask;
  int32_t exact_broad_phase;
  int32_t fused_kernel;  /* > 0: a handle from vmas_b200_register_step_kernel (direct mode only) */
  const VmasStepProgram* program;
  const int32_t* columns;
  int32_t n_rows, width;
  float* obs_out;
  /* 3 */
  const VmasCopySegment* segs;
  const int32_t* seg_block;
  int32_t n_segs, n_out_blocks;
  void* out_blocks[VMAS_MAX_OUT_BLOCKS];
  /* direct mode: results written straight into the caller's fresh blocks instead of being copied there.
   * obs_block >= 0: the observation rows go to out_blocks[obs_block] + obs_offset (not to `obs_out`);
   * mirror i: program buffer slot mirror_slot[i] (the target of a STORE instruction the caller appended for
   * one of its result leaves) is out_blocks[mirror_block[i]] + mirror_offset[i] in this step. */
  int32_t obs_block, n_mirrors;
  size_t obs_offset;
  /* != 0 (direct mode with `fused_kernel`): the whole step goes out as ONE launch if the kernel has the
   * ingest prologue for these agents (continuous holonomic actions) and the batch fits the GPU at once (a
   * masked world's broad phase needs a grid-wide barrier per substep; `mask` must then hold
   * substeps x ((n_masked + 31) / 32 + 2) zeroed words); otherwise the launches above are issued. */
  int32_t ingest_in_kernel;
  /* what the post stage writes to out_blocks[obs_block] (obs_block >= 0; rows going to `obs_out` are fp32):
   * VMAS_DTYPE_F32, or VMAS_DTYPE_F16 / VMAS_DTYPE_BF16 — each value rounded to nearest even; a `fused_kernel`
   * must then have been compiled for that type */
  int32_t obs_dtype;
  int32_t mirror_slot[VMAS_PROG_MAX_BUFFERS];
  int32_t mirror_block[VMAS_PROG_MAX_BUFFERS];
  size_t mirror_offset[VMAS_PROG_MAX_BUFFERS];
  /* NULL, or n_segs kinds of the hand-out segments as vmas_b200_copy_buffers_convert takes them */
  const int32_t* seg_kind;
} VmasEnvStep;
int vmas_b200_env_step(const VmasEnvStep* step, void* cuda_stream);

/* The broad-phase pass alone: ORs bit i of `mask` if masked item i is within range in any env. */
int vmas_b200_broad_phase(const VmasWorldConfig* cfg, const VmasPlanTables* tb, const VmasState* st,
                          uint32_t* mask, void* cuda_stream);

/*
 * Device-side episode reset (SURVEY §8(f)-4).  Env selection, for both calls:
 *   env_index >= 0            that env only (Environment.reset_at(i), ref environment.py:229-252)
 *   env_index < 0, mask NULL  every env      (Environment.reset,     ref environment.py:204-227)
 *   env_index < 0, mask       every env with env_mask[env] != 0 (device uint8[B]) — a batched
 *                             reset of the envs that are done, which the reference does one
 *                             reset_at() at a time
 *
 * vmas_b200_reset_state: World.reset(env_index) (ref core.py:1179-1181 -> EntityState._reset
 * core.py:286-296, 371-383): zeroes pos, vel, rot, ang_vel of every entity and force, torque of
 * every agent in the selected envs, one launch.  `reset_count` (device int32[B] or NULL) is the
 * per-env episode number; it is incremented for the selected envs.
 */
int vmas_b200_reset_state(const VmasWorldConfig* cfg, const VmasState* st, int32_t env_index,
                          const uint8_t* env_mask, int32_t* reset_count, void* cuda_stream);

/*
 * ScenarioUtils.spawn_entities_randomly / find_random_pos_for_entity (ref utils.py:241-319):
 * per selected env, draws `n_spawn` positions one after the other, each uniform in
 * [x_lo, x_hi] x [y_lo, y_hi] and re-drawn until it is at least `min_dist` away from every
 * occupied point (the listed slab entities, the extra `occupied` points, and the positions drawn
 * earlier in this call).  One thread per env, no host synchronisation (the reference loops in
 * python with one torch.any() sync per attempt).
 *
 * Random numbers are Philox4x32-10 with counter (env_offset + env, reset_count[env], stream_id,
 * i << 26 | attempt / 2) and key `seed`: the position of draw i of an env is independent of which other
 * envs are selected in the launch (masked reset == one reset_at per env, bit for bit), and
 * oracle/reset.py reproduces it on the CPU.  A draw that still overlaps after `max_tries`
 * attempts keeps its last proposal and `*status` is incremented (the reference would keep looping).
 */
#define VMAS_MAX_SPAWN 64
typedef struct VmasSpawn {
  int32_t n_spawn;
  int32_t entity[VMAS_MAX_SPAWN];          /* slab entity that receives draw i, or -1: only written to `out` */
  int32_t n_occupied_entities;
  int32_t occupied_entity[VMAS_MAX_SPAWN]; /* slab entities (already placed) to keep away from */
  const float* occupied;                   /* device fp32 [., n_occupied, 2] further occupied points, or NULL */
  int32_t n_occupied;
  int32_t max_tries;                       /* attempts per draw, in [1, 2^27] */
  int64_t occupied_env_stride;             /* elements between consecutive envs of `occupied`; 0: shared by all envs */
  float* out;                              /* device fp32 [B, n_spawn, 2] or NULL: the positions drawn (selected envs only) */
  float min_dist, x_lo, x_hi, y_lo, y_hi;
  int32_t env_index;
  const uint8_t* env_mask;
  uint64_t seed;
  uint32_t stream_id;                      /* which spawn call since the env's last reset this is */
  uint32_t env_offset;                     /* index of this slab's env 0 in the whole job (batch_dim sharded over
                                              GPUs): counters use env + env_offset, so a shard draws what the
                                              unsharded job draws for the same envs */
  const int32_t* reset_count;              /* device int32[B] or NULL (= 0) */
  int32_t* status;                         /* device int32[1] or NULL */
} VmasSpawn;

int vmas_b200_spawn_entities(const VmasWorldConfig* cfg, const VmasState* st, const VmasSpawn* spawn,
                             void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* VMAS_B200_H */
