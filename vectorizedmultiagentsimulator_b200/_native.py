"""ctypes binding of the C-ABI library ``libvmas_b200.so`` (``include/vmas_b200.h``).

The library is built in-tree by :func:`build` (``nvcc -gencode arch=compute_90a,code=sm_90a``)
and loaded by :func:`load`, which fails loudly if it is missing: there is no fallback path.
PyTorch only provides device memory and the current stream; every kernel is this library's.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import weakref
from typing import Optional

import numpy as np
import torch

from .simulator import plan as P

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(_ROOT, "include")
#: Arithmetic of the kernels.  "exact" (default): every multiply / add rounds on its own and division
#: and square root are IEEE — the reference's eager op chain, reproduced to ~1e-6.  "fast": the same
#: sources built with FMA contraction and approximate division / square root (<= 2 ulp each; sin,
#: cos, exp, log stay precise) — still inside the 1e-4 relative contract of the north star for
#: worlds without joints, for 30-36 % fewer instructions in the substep kernels (DESIGN §7).  It is a
#: separate library so the two can be compared side by side: VMAS_B200_ARITH=fast.
ARITH = os.environ.get("VMAS_B200_ARITH", "exact")
assert ARITH in ("exact", "fast"), f"VMAS_B200_ARITH must be 'exact' or 'fast', got {ARITH!r}"


def lib_path_for(arith: str) -> str:
    return os.path.join(_HERE, "libvmas_b200.so" if arith == "exact" else "libvmas_b200_fast.so")


LIB_PATH = os.environ.get("VMAS_B200_LIB") or lib_path_for(ARITH)
SOURCES = [os.path.join(CSRC, "vmas_b200.cu")]
GENERATED = os.path.join(CSRC, "generated", "specializations.cuh")
HEADERS = [
    os.path.join(CSRC, "geometry.cuh"),
    os.path.join(CSRC, "generic_step.cuh"),
    os.path.join(CSRC, "query.cuh"),
    os.path.join(CSRC, "ingest.cuh"),
    os.path.join(CSRC, "rays.cuh"),
    os.path.join(CSRC, "spec_kernel.cuh"),
    os.path.join(CSRC, "spec_tile_kernel.cuh"),
    os.path.join(CSRC, "reset.cuh"),
    os.path.join(INCLUDE, "vmas_b200.h"),
    GENERATED,
]

ARITH_FLAGS = {
    "exact": ["-fmad=false"],  # every mul/add rounds on its own, like the reference's eager op chain
    "fast": ["-fmad=true", "-prec-div=false", "-prec-sqrt=false"],
}
NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-O3",
    "-lineinfo",
    "-DSPEC_MIN_BLOCKS=8",  # <= 128 registers for the specialised kernels: 16 warps/SM
    "-std=c++17",
    "-Xcompiler",
    "-fPIC",
    "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libvmas_b200.so")


def needs_build(lib_path: Optional[str] = None) -> bool:
    lib_path = lib_path or LIB_PATH
    if not os.path.exists(lib_path) or not os.path.exists(GENERATED):
        return True
    built = os.path.getmtime(lib_path)
    return any(os.path.getmtime(f) > built for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False, arith: Optional[str] = None) -> str:
    """Compile the CUDA sources for sm_90a into ``libvmas_b200.so`` (``arith="fast"``:
    ``libvmas_b200_fast.so``) next to this file.  Default: the variant this process loads."""
    from . import codegen

    codegen.generate(GENERATED)  # constexpr world tables for the specialised kernels (no-op if unchanged)
    lib_path = LIB_PATH if arith is None else lib_path_for(arith)
    if not force and not needs_build(lib_path):
        return lib_path
    extra = os.environ.get("VMAS_B200_NVCC_EXTRA", "").split()
    flags = NVCC_FLAGS + ARITH_FLAGS[arith or ARITH]
    cmd = [_nvcc()] + flags + extra + ["-I", INCLUDE, "-I", CSRC, "-o", lib_path] + SOURCES
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{proc.stdout}\n{proc.stderr}")
    if verbose:
        print(proc.stderr)
    return lib_path


# ---------------------------------------------------------------------------------------------
# ctypes mirrors of the header structs
# ---------------------------------------------------------------------------------------------
class WorldConfig(C.Structure):
    _fields_ = [
        ("batch_dim", C.c_int32),
        ("n_entities", C.c_int32),
        ("n_agents", C.c_int32),
        ("n_items", C.c_int32),
        ("n_joints", C.c_int32),
        ("n_masked", C.c_int32),
        ("substeps", C.c_int32),
        ("has_x_semidim", C.c_int32),
        ("has_y_semidim", C.c_int32),
        ("has_world_gravity", C.c_int32),
        ("sub_dt", C.c_float),
        ("x_semidim", C.c_float),
        ("y_semidim", C.c_float),
        ("collision_force", C.c_float),
        ("joint_force", C.c_float),
        ("torque_constraint_force", C.c_float),
        ("contact_margin", C.c_float),
        ("gravity_x", C.c_float),
        ("gravity_y", C.c_float),
    ]


class PlanTablesC(C.Structure):
    _fields_ = [
        ("ent_f32", C.c_void_p),
        ("ent_i32", C.c_void_p),
        ("item_f32", C.c_void_p),
        ("item_i32", C.c_void_p),
        ("inc_off", C.c_void_p),
        ("inc", C.c_void_p),
        ("sched", C.c_void_p),
        ("masked_items", C.c_void_p),
        ("joint_rot", C.c_void_p),
        ("ent_gravity", C.c_void_p),
        ("n_rounds", C.c_int32),
        ("group", C.c_int32),
        ("ents_per_lane", C.c_int32),
        ("specialization", C.c_int32),
        ("env_order", C.c_void_p),
        ("env_signature", C.c_void_p),
    ]


class StateC(C.Structure):
    _fields_ = [
        ("pos", C.c_void_p),
        ("vel", C.c_void_p),
        ("rot", C.c_void_p),
        ("ang_vel", C.c_void_p),
        ("force", C.c_void_p),
        ("torque", C.c_void_p),
    ]


MAX_INGEST_AGENTS = 16
MAX_ACTION_SIZE = 8


class AgentActionsC(C.Structure):
    _fields_ = [
        ("actions", C.c_void_p),
        ("u", C.c_void_p),
        ("action_size", C.c_int32),
        ("agent_index", C.c_int32),
        ("dynamics", C.c_int32),
        ("entity_index", C.c_int32),
        ("u_range", C.c_float * MAX_ACTION_SIZE),
        ("u_multiplier", C.c_float * MAX_ACTION_SIZE),
        ("dyn_params", C.c_float * 8),
        ("dyn_state", C.c_void_p),
        ("action_kind", C.c_int32),
        ("nvec", C.c_int32 * MAX_ACTION_SIZE),
    ]


ACT_CONTINUOUS, ACT_DISCRETE, ACT_MULTIDISCRETE = 0, 1, 2


DYN_NONE, DYN_HOLONOMIC, DYN_HOLONOMIC_ROT, DYN_FORWARD, DYN_ROTATION, DYN_DIFF_DRIVE, DYN_BICYCLE, DYN_DRONE = -1, 0, 1, 2, 3, 4, 5, 6


MAX_SPAWN = 64
GROUP_TILE = -8  # VMAS_GROUP_TILE
GROUP_BLOCK = -16  # VMAS_GROUP_BLOCK
#: entities per env the CUDA backend steps (VMAS_BLOCK_MAX_ENTITIES: the block-per-env kernel's limit)
MAX_ENTITIES = 1024
#: opt-in shared memory per block of sm_90 (227 KB), taken for a device without properties (``cpu``)
SM90_SHARED_OPTIN = 232448
TPE_FIELDS, TPE_MIN_BLOCK = 13, 32  # step_tpe_kernel: [13 fields][E][BLOCK] fp32, BLOCK = 64 or 32
#: env scheduling of the specialised thread-per-env kernel: the envs are re-sorted by their contact
#: signature every this many World.step calls (0 = off: thread t always steps env t).  OFF by default:
#: it halves the warp-instructions (1.8 k per 32 envs at 31 of 32 lanes active) but the scattered rows
#: leave the kernel latency-bound — measured slower on real roll-out states
ENV_REORDER_EVERY = int(os.environ.get("VMAS_B200_ENV_REORDER_EVERY", "0"))
ENV_REORDER_MIN_BATCH = 1024  # below this there is nothing to gain from grouping
ENV_REORDER_CHUNK = int(os.environ.get("VMAS_B200_ENV_REORDER_CHUNK", "2048"))  # envs sorted together
#: what mapping="auto" picks for a specialised world that has both kernels
DEFAULT_SPEC_MAPPING = os.environ.get("VMAS_B200_SPEC_MAPPING", "specialized")
#: the values of ``DeviceTables(mapping=...)`` / ``VMAS_B200_MAPPING``
MAPPINGS = ("auto", "specialized", "tile", "thread_per_env", "lanes_per_env", "block_per_env")


class SpawnC(C.Structure):
    """``VmasSpawn`` (include/vmas_b200.h)."""

    _fields_ = [
        ("n_spawn", C.c_int32),
        ("entity", C.c_int32 * MAX_SPAWN),
        ("n_occupied_entities", C.c_int32),
        ("occupied_entity", C.c_int32 * MAX_SPAWN),
        ("occupied", C.c_void_p),
        ("n_occupied", C.c_int32),
        ("max_tries", C.c_int32),
        ("occupied_env_stride", C.c_int64),
        ("out", C.c_void_p),
        ("min_dist", C.c_float),
        ("x_lo", C.c_float),
        ("x_hi", C.c_float),
        ("y_lo", C.c_float),
        ("y_hi", C.c_float),
        ("env_index", C.c_int32),
        ("env_mask", C.c_void_p),
        ("seed", C.c_uint64),
        ("stream_id", C.c_uint32),
        ("env_offset", C.c_uint32),
        ("reset_count", C.c_void_p),
        ("status", C.c_void_p),
    ]


EXPORTS = [
    "vmas_b200_abi_version",
    "vmas_b200_last_error",
    "vmas_b200_num_specializations",
    "vmas_b200_find_specialization",
    "vmas_b200_specialization_name",
    "vmas_b200_specialization_has_tile",
    "vmas_b200_register_specialization",
    "vmas_b200_world_step",
    "vmas_b200_world_step_params",
    "vmas_b200_world_substeps",
    "vmas_b200_world_step_timed",
    "vmas_b200_cast_rays",
    "vmas_b200_pair_query",
    "vmas_b200_point_query",
    "vmas_b200_broad_phase",
    "vmas_b200_ingest_actions",
    "vmas_b200_ingest_actions_broad_phase",
    "vmas_b200_velocity_controller",
    "vmas_b200_cast_rays_batched",
    "vmas_b200_pair_query_batched",
    "vmas_b200_gather_observations",
    "vmas_b200_gather_observations_buffers",
    "vmas_b200_distance_shaping",
    "vmas_b200_post_step",
    "vmas_b200_copy_buffers",
    "vmas_b200_copy_buffers_convert",
    "vmas_b200_env_step",
    "vmas_b200_register_step_kernel",
    "vmas_b200_graph_num_nodes",
    "vmas_b200_build_env_order",
    "vmas_b200_set_l2_fetch_granularity",
    "vmas_b200_reset_state",
    "vmas_b200_spawn_entities",
]

_lib = None


def load():
    """Load the built library (never builds implicitly: run ``build()`` first)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(needs nvcc). vectorizedmultiagentsimulator_b200 has no CPU / torch fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise RuntimeError(f"{LIB_PATH} does not export {name}; rebuild it")
    lib.vmas_b200_abi_version.restype = C.c_int
    lib.vmas_b200_last_error.restype = C.c_char_p
    p_cfg, p_tb, p_st = C.POINTER(WorldConfig), C.POINTER(PlanTablesC), C.POINTER(StateC)
    lib.vmas_b200_world_step.argtypes = [p_cfg, p_tb, p_st, C.c_void_p, C.c_int, C.c_void_p]
    lib.vmas_b200_world_step_params.argtypes = [p_cfg, p_tb, C.c_void_p, p_st, C.c_void_p, C.c_int, C.c_void_p]
    lib.vmas_b200_world_substeps.argtypes = [
        p_cfg, p_tb, p_st, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p
    ]
    lib.vmas_b200_world_step_timed.argtypes = [
        p_cfg, p_tb, p_st, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_cast_rays.argtypes = [
        p_cfg, p_tb, p_st, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
        C.c_float, C.c_void_p, C.c_void_p,
    ]
    lib.vmas_b200_pair_query.argtypes = [
        p_cfg, p_tb, p_st, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_point_query.argtypes = [p_cfg, p_tb, p_st, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.vmas_b200_broad_phase.argtypes = [p_cfg, p_tb, p_st, C.c_void_p, C.c_void_p]
    lib.vmas_b200_cast_rays_batched.argtypes = [
        p_cfg, p_tb, p_st, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
    ]
    lib.vmas_b200_gather_observations.argtypes = [
        p_cfg, p_st, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_gather_observations_buffers.argtypes = [
        p_cfg, p_st, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p
    ]
    lib.vmas_b200_distance_shaping.argtypes = [
        p_cfg, p_st, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_pair_query_batched.argtypes = [
        p_cfg, p_tb, p_st, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_ingest_actions.argtypes = [
        p_cfg, p_st, C.POINTER(AgentActionsC), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_ingest_actions_broad_phase.argtypes = [
        p_cfg, p_tb, p_st, C.POINTER(AgentActionsC), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_reset_state.argtypes = [p_cfg, p_st, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.vmas_b200_spawn_entities.argtypes = [p_cfg, p_st, C.POINTER(SpawnC), C.c_void_p]
    lib.vmas_b200_copy_buffers.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.vmas_b200_copy_buffers_convert.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.vmas_b200_post_step.argtypes = [
        p_cfg, p_tb, p_st, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p
    ]
    lib.vmas_b200_velocity_controller.argtypes = [
        p_cfg, p_st, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
        C.c_float, C.c_float, C.c_void_p,
    ]
    lib.vmas_b200_env_step.argtypes = [C.c_void_p, C.c_void_p]
    lib.vmas_b200_graph_num_nodes.argtypes = [C.c_void_p]
    lib.vmas_b200_register_step_kernel.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.vmas_b200_build_env_order.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.vmas_b200_set_l2_fetch_granularity.argtypes = [C.c_int32]
    lib.vmas_b200_find_specialization.argtypes = [C.c_uint64]
    lib.vmas_b200_specialization_name.argtypes = [C.c_int]
    lib.vmas_b200_specialization_has_tile.argtypes = [C.c_int]
    lib.vmas_b200_register_specialization.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]
    for name in EXPORTS[2:]:
        getattr(lib, name).restype = C.c_int
    lib.vmas_b200_specialization_name.restype = C.c_char_p
    if lib.vmas_b200_abi_version() != 2:
        raise RuntimeError("libvmas_b200.so ABI version mismatch; rebuild it")
    _lib = lib
    return lib


_restore_device = None  # the caller's current device while a launch on another GPU is in flight


def _check(lib, rc: int) -> int:
    """Every launch wrapper ends here: error check, and the caller's current CUDA device is put back
    if ``_stream`` had to switch it (a world on cuda:1 must not leave the process on cuda:1)."""
    global _restore_device
    if _restore_device is not None:
        torch.cuda.set_device(_restore_device)
        _restore_device = None
    if rc < 0:
        raise RuntimeError(f"vmas_b200: {lib.vmas_b200_last_error().decode()}")
    return rc


def _stream(device) -> int:
    # kernels launch on the calling thread's current device: make it the world's device for the
    # duration of the call (``_check`` restores the caller's)
    global _restore_device
    index = device.index
    current = torch.cuda.current_device()
    if current != index:
        if _restore_device is None:
            _restore_device = current
        torch.cuda.set_device(device)
    return _raw_stream(index)


try:  # the raw handle of the current stream without building a torch.cuda.Stream object
    _raw_stream = torch._C._cuda_getCurrentRawStream
except AttributeError:  # pragma: no cover

    def _raw_stream(index: int) -> int:
        return torch.cuda.current_stream(index).cuda_stream


# ---------------------------------------------------------------------------------------------
# device-resident plan
# ---------------------------------------------------------------------------------------------
def lane_layout(n_entities: int):
    """(lanes per env, entities per lane) for the substep kernel."""
    if n_entities <= 8:
        return 8, 1
    if n_entities <= 16:
        return 16, 1
    if n_entities <= 32:
        return 32, 1
    if n_entities <= 64:
        return 32, 2
    if n_entities <= 128:
        return 32, 4
    raise NotImplementedError(f"{n_entities} entities per env exceed the kernel's limit of 128")


def shared_optin_bytes(device) -> int:
    """Opt-in shared memory per block of ``device`` (the sm_90 value for a non-CUDA device)."""
    device = torch.device(device)
    if device.type != "cuda":
        return SM90_SHARED_OPTIN
    return int(torch.cuda.get_device_properties(device).shared_memory_per_block_optin)


def tpe_fits(tables: P.PlanTables, device) -> bool:
    """Whether the thread-per-env kernel's smallest block (32 envs) holds an env's state and the mask words."""
    state = TPE_FIELDS * tables.desc.n_entities * TPE_MIN_BLOCK * 4
    return state + 4 * ((tables.n_masked + 31) // 32) <= shared_optin_bytes(device)


def make_config(tables: P.PlanTables, batch_dim: Optional[int] = None) -> WorldConfig:
    d = tables.desc
    cfg = WorldConfig()
    cfg.batch_dim = d.batch_dim if batch_dim is None else batch_dim
    cfg.n_entities = d.n_entities
    cfg.n_agents = d.n_agents
    cfg.n_items = len(d.items)
    cfg.n_joints = tables.n_joints
    cfg.n_masked = tables.n_masked
    cfg.substeps = d.substeps
    cfg.has_x_semidim = int(d.x_semidim is not None)
    cfg.has_y_semidim = int(d.y_semidim is not None)
    cfg.has_world_gravity = int(any(g != 0.0 for g in d.gravity))
    cfg.sub_dt = d.dt / d.substeps
    cfg.x_semidim = d.x_semidim or 0.0
    cfg.y_semidim = d.y_semidim or 0.0
    cfg.collision_force = d.collision_force
    cfg.joint_force = d.joint_force
    cfg.torque_constraint_force = d.torque_constraint_force
    cfg.contact_margin = d.contact_margin
    cfg.gravity_x, cfg.gravity_y = d.gravity
    return cfg


class DeviceTables:
    """The plan tables uploaded to one GPU, plus the ctypes structs pointing at them."""

    def __init__(self, tables: P.PlanTables, world, device, mapping: Optional[str] = None):
        self.tables = tables
        self.device = torch.device(device)
        desc = tables.desc
        mapping = mapping or os.environ.get("VMAS_B200_MAPPING", "auto")
        if mapping not in MAPPINGS:
            raise ValueError(f"unknown mapping {mapping!r}: expected one of {', '.join(MAPPINGS)}")
        if desc.n_entities > MAX_ENTITIES:
            raise NotImplementedError(
                f"{desc.n_entities} entities per env exceed the CUDA backend's limit of {MAX_ENTITIES}"
            )
        self.specialization = -1
        # specialised worlds have two kernels: "specialized" = one thread per env (step_spec_kernel),
        # "tile" = a warp per 32 envs with the narrow phase compacted (step_tile_kernel; not for
        # worlds with joints).  "auto" takes DEFAULT_SPEC_MAPPING where the world has it.
        if mapping in ("auto", "specialized", "tile"):
            from . import codegen

            lib = load()
            self.specialization = lib.vmas_b200_find_specialization(codegen.world_hash(desc))
            if self.specialization < 0:
                if mapping != "auto":
                    raise RuntimeError("no ahead-of-time specialisation of this world in libvmas_b200.so")
                mapping = "thread_per_env" if tpe_fits(tables, self.device) else "block_per_env"
            else:
                has_tile = bool(lib.vmas_b200_specialization_has_tile(self.specialization))
                if mapping == "tile" and not has_tile:
                    raise RuntimeError("this world's specialisation has no tile kernel (joints / too many work items)")
                if mapping == "auto":
                    mapping = "tile" if (has_tile and DEFAULT_SPEC_MAPPING == "tile") else "specialized"
        self.mapping = mapping
        if mapping in ("thread_per_env", "specialized", "tile", "block_per_env"):
            group = {"tile": GROUP_TILE, "block_per_env": GROUP_BLOCK}.get(mapping, 1)
            self.group, self.ents_per_lane = group, desc.n_entities
            sched = np.zeros((0, 1), np.int32)
        else:
            self.group, self.ents_per_lane = lane_layout(desc.n_entities)
            sched, _ = tables.schedule(self.group)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        self.ent_f32 = up(tables.ent_f32)
        self.ent_i32 = up(tables.ent_i32)
        self.item_f32 = up(tables.item_f32)
        self.item_i32 = up(tables.item_i32)
        self.inc_off = up(tables.inc_off)
        self.inc = up(tables.inc)
        self.sched = up(sched if sched.size else np.full((1, max(self.group, 1)), -1, np.int32))
        self.masked_items = up(tables.masked_items)
        B = desc.batch_dim if world is None else world.batch_dim
        needs_rot = any(it["kind"] == P.K_JOINT and not it["rotate"] for it in desc.items)
        self.joint_rot = (
            torch.zeros(B, max(tables.n_joints, 1), dtype=torch.float32, device=self.device)
            if needs_rot
            else None
        )
        if self.joint_rot is not None:
            # every non-rotating joint reads its angle per env; scalar ones are broadcast here
            self.item_i32[: tables.n_joints, 3] |= P.IFLAG_JOINT_ROT_PER_ENV
            for k, it in enumerate(desc.items[: tables.n_joints]):
                if not it["rotate"] and it["fixed_rotation"] is not None:
                    self.joint_rot[:, k] = float(it["fixed_rotation"])
        self.gravity_entities = [i for i, e in enumerate(desc.entities) if e.get("gravity_per_env")]
        self.ent_gravity = (
            torch.zeros(B, desc.n_entities, 2, dtype=torch.float32, device=self.device)
            if self.gravity_entities
            else None
        )
        # per-env mass / friction coefficients: [B, E, EP_COLS], the rows of flagged entities written before each
        # step (CudaBackend._sync_entity_params)
        self.param_entities = [
            i for i, e in enumerate(desc.entities)
            if e.get("mass_per_env") or e.get("lin_fric_per_env") or e.get("ang_fric_per_env")
        ]
        self.ent_params = (
            torch.zeros(B, desc.n_entities, P.EP_COLS, dtype=torch.float32, device=self.device)
            if self.param_entities
            else None
        )
        words = (tables.n_masked + 31) // 32
        # (+ the kernels' arrival counters; the one-kernel step keeps a mask per substep)
        self.mask = torch.zeros(max(1, int(tables.desc.substeps)) * (words + 2), dtype=torch.int32, device=self.device)
        self.n_rounds = int(sched.shape[0])

        self.cfg = make_config(tables, B)
        tb = PlanTablesC()
        tb.ent_f32 = self.ent_f32.data_ptr()
        tb.ent_i32 = self.ent_i32.data_ptr()
        tb.item_f32 = self.item_f32.data_ptr()
        tb.item_i32 = self.item_i32.data_ptr()
        tb.inc_off = self.inc_off.data_ptr()
        tb.inc = self.inc.data_ptr()
        tb.sched = self.sched.data_ptr()
        tb.masked_items = self.masked_items.data_ptr()
        tb.joint_rot = self.joint_rot.data_ptr() if self.joint_rot is not None else None
        tb.ent_gravity = self.ent_gravity.data_ptr() if self.ent_gravity is not None else None
        tb.n_rounds = self.n_rounds
        tb.group = self.group
        tb.ents_per_lane = self.ents_per_lane
        tb.specialization = self.specialization
        # env scheduling (specialised thread-per-env kernel only): identity order until the first
        # re-ordering, so a captured CUDA graph already reads the table it will keep reading
        self.env_order = self.env_signature = None
        if self.mapping == "specialized" and ENV_REORDER_EVERY > 0 and B >= ENV_REORDER_MIN_BATCH:
            self.env_order = torch.arange(B, dtype=torch.int32, device=self.device)
            self.env_signature = torch.zeros(B, dtype=torch.int32, device=self.device)
            tb.env_order = self.env_order.data_ptr()
            tb.env_signature = self.env_signature.data_ptr()
        self.tb = tb
        self._state_key = None
        self._state_ref = None
        self._state = None

    def state_struct(self, slab) -> StateC:
        # a slab's tensors are allocated once: the struct is cached per (live) slab object
        ref = self._state_ref
        if ref is not None and ref() is slab:
            return self._state
        self._state_ref = weakref.ref(slab)
        key = tuple(t.data_ptr() for t in slab.tensors())
        if key != self._state_key:
            for t in slab.tensors():
                assert t.is_contiguous() and t.dtype == torch.float32 and t.device == self.device
            st = StateC()
            st.pos, st.vel, st.rot, st.ang_vel, st.force, st.torque = key
            self._state, self._state_key = st, key
        return self._state


# ---------------------------------------------------------------------------------------------
# call wrappers
# ---------------------------------------------------------------------------------------------
def world_step(lib, dt: DeviceTables, slab, exact_broad_phase: bool = True, events=None) -> int:
    """One World.step.  ``events``: optional (begin, end) torch.cuda.Event pair (timing enabled)
    recorded around the substep kernel(s) only."""
    st = dt.state_struct(slab)
    if dt.ent_params is not None:
        if events is not None:
            events[0].record()
        rc = lib.vmas_b200_world_step_params(
            C.byref(dt.cfg), C.byref(dt.tb), dt.ent_params.data_ptr(), C.byref(st), dt.mask.data_ptr(),
            int(exact_broad_phase), _stream(dt.device),
        )
        if events is not None:
            events[1].record()
    elif events is None:
        rc = lib.vmas_b200_world_step(
            C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), dt.mask.data_ptr(), int(exact_broad_phase),
            _stream(dt.device),
        )
    else:
        # torch creates the underlying cudaEvent lazily on first record(): force creation
        for ev in events:
            if not ev.cuda_event:
                ev.record()
        rc = lib.vmas_b200_world_step_timed(
            C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), dt.mask.data_ptr(), int(exact_broad_phase),
            _stream(dt.device), events[0].cuda_event, events[1].cuda_event,
        )
    return _check(lib, rc)


def build_env_order(lib, dt: DeviceTables) -> int:
    """Re-sorts ``dt.env_order`` by the contact signatures the last step recorded (one launch)."""
    if dt.env_order is None:
        return 0
    rc = lib.vmas_b200_build_env_order(
        dt.env_signature.data_ptr(), int(dt.env_order.shape[0]), dt.env_order.data_ptr(), ENV_REORDER_CHUNK,
        _stream(dt.device),
    )
    return _check(lib, rc)


def world_substeps(lib, dt: DeviceTables, slab, first: int, n: int, exact_broad_phase: bool = True) -> int:
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_world_substeps(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), dt.mask.data_ptr(), int(exact_broad_phase), first, n,
        _stream(dt.device),
    )
    return _check(lib, rc)


def cast_rays(lib, dt: DeviceTables, slab, src, targets, n_targets, angles, add_rot_of, max_range, out) -> int:
    st = dt.state_struct(slab)
    assert angles.is_contiguous() and out.is_contiguous() and angles.dtype == torch.float32
    rc = lib.vmas_b200_cast_rays(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), int(src), targets.data_ptr(), int(n_targets),
        angles.data_ptr(), int(angles.shape[-1]), -1 if add_rot_of is None else int(add_rot_of),
        float(max_range), out.data_ptr(), _stream(dt.device),
    )
    return _check(lib, rc)


def pair_query(lib, dt: DeviceTables, slab, a: int, b: int, mode: int, out) -> int:
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_pair_query(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), a, b, mode, out.data_ptr(), _stream(dt.device)
    )
    return _check(lib, rc)


def point_query(lib, dt: DeviceTables, slab, entity: int, point, out) -> int:
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_point_query(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), entity, point.data_ptr(), out.data_ptr(), _stream(dt.device)
    )
    return _check(lib, rc)


def broad_phase(lib, dt: DeviceTables, slab) -> int:
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_broad_phase(C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), dt.mask.data_ptr(), _stream(dt.device))
    return _check(lib, rc)


def ingest_actions(lib, dt: DeviceTables, slab, agents_c, n: int, clamp: bool, bad_flag, steps=None, broad_phase=False) -> int:
    """``agents_c``: a ctypes array of AgentActionsC whose pointers are already filled in; ``steps``: the
    environment's fp32 ``[B]`` step counter to increment in the same launch, or None; ``broad_phase``: also
    build the broad-phase mask of the coming step's first substep (the next ``world_step`` is then called
    with ``exact_broad_phase=2``)."""
    st = dt.state_struct(slab)
    if broad_phase:
        rc = lib.vmas_b200_ingest_actions_broad_phase(
            C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), agents_c, n, int(clamp),
            None if bad_flag is None else bad_flag.data_ptr(), None if steps is None else steps.data_ptr(),
            dt.mask.data_ptr(), _stream(dt.device),
        )
        return _check(lib, rc)
    rc = lib.vmas_b200_ingest_actions(
        C.byref(dt.cfg), C.byref(st), agents_c, n, int(clamp),
        None if bad_flag is None else bad_flag.data_ptr(), None if steps is None else steps.data_ptr(),
        _stream(dt.device),
    )
    return _check(lib, rc)


def cast_rays_batched(
    lib, dt: DeviceTables, slab, src, target_off, targets, angles, max_range, n_rays, out, out_offsets=None,
    out_env_stride: int = 0, flags: int = 0,
) -> int:
    """``out``: dense [Q, B, R] block, or (with ``out_offsets`` int64[Q] and ``out_env_stride``)
    any fp32 tensor the readings are scattered into (columns of an observation block)."""
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_cast_rays_batched(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), int(src.shape[0]), src.data_ptr(), target_off.data_ptr(),
        targets.data_ptr(), angles.data_ptr(), max_range.data_ptr(), int(n_rays), out.data_ptr(),
        out_offsets.data_ptr() if out_offsets is not None else None, int(out_env_stride), int(flags),
        _stream(dt.device),
    )
    return _check(lib, rc)


def velocity_controller(lib, dt: DeviceTables, slab, entity: int, u, accum, prev, gain, inv_ti, td, step_dt, windup, mass) -> int:
    """PID force from a velocity target, in place on ``u`` [B, 2] (see include/vmas_b200.h)."""
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_velocity_controller(
        C.byref(dt.cfg), C.byref(st), int(entity), u.data_ptr(), accum.data_ptr(), prev.data_ptr(), float(gain),
        float(inv_ti), float(td), float(step_dt), float(windup), float(mass), _stream(dt.device),
    )
    return _check(lib, rc)


PROG_MAX_INSTR, PROG_MAX_BUFFERS = 64, 32


class ProgInstrC(C.Structure):
    _fields_ = [("op", C.c_uint8), ("dst", C.c_uint8), ("a", C.c_uint8), ("b", C.c_uint8), ("arg", C.c_int32), ("imm", C.c_float)]


class StepProgramC(C.Structure):
    _fields_ = [
        ("n_instr", C.c_int32),
        ("reserved", C.c_int32),
        ("instr", ProgInstrC * PROG_MAX_INSTR),
        ("buffers", C.c_void_p * PROG_MAX_BUFFERS),
    ]


def post_step(lib, dt: DeviceTables, slab, program, columns, n_rows: int, width: int, out) -> int:
    """The scenario's step program and (optionally) the observation gather in one launch."""
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_post_step(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), C.byref(program) if program is not None else None,
        None if columns is None else columns.data_ptr(), int(n_rows), int(width),
        None if out is None else out.data_ptr(), _stream(dt.device),
    )
    return _check(lib, rc)


class CopySegmentC(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("bytes", C.c_size_t)]


MAX_COPY_SEGMENTS = 64
#: element types of observation results (``VMAS_DTYPE_*``): what a converting copy segment writes, what the post
#: stage stores; fp32 is a plain copy
DTYPE_F32, DTYPE_F16, DTYPE_BF16 = 0, 1, 2
DTYPE_CODES = {torch.float32: DTYPE_F32, torch.float16: DTYPE_F16, torch.bfloat16: DTYPE_BF16}


def copy_buffers(lib, device, pairs) -> int:
    """``pairs``: [(src tensor, dst tensor)] of equal byte size, contiguous, on ``device``: one launch
    per ``MAX_COPY_SEGMENTS`` of them."""
    n = 0
    for lo in range(0, len(pairs), MAX_COPY_SEGMENTS):
        chunk = pairs[lo : lo + MAX_COPY_SEGMENTS]
        segs = (CopySegmentC * len(chunk))()
        for seg, (src, dst) in zip(segs, chunk):
            seg.src, seg.dst, seg.bytes = src.data_ptr(), dst.data_ptr(), src.numel() * src.element_size()
        n += _check(lib, lib.vmas_b200_copy_buffers(segs, len(chunk), _stream(device)))
    return n


def _segment_kinds(items, block_kinds):
    """``int32[n]`` kinds of the copy segments ``items`` = [(source, block, offset)] (``block_kinds[b]``: what
    block ``b`` receives, ``DTYPE_F32`` = a plain copy), or None when every segment is a plain copy."""
    if not block_kinds or not any(block_kinds[block] for _, block, _ in items):
        return None
    kinds = (C.c_int32 * len(items))()
    for k, (src, block, _) in enumerate(items):
        kinds[k] = block_kinds[block]
        assert not kinds[k] or src.dtype == torch.float32, "a converting copy reads fp32"
    return kinds


class CopyPlan:
    """A fixed list of copies whose SOURCES never move (the buffers a captured step writes) into
    destination blocks that are allocated anew every step: sources, sizes and destination offsets are
    marshalled once, a run only adds the fresh base addresses."""

    def __init__(self, items, block_kinds=None):
        """``items``: [(source tensor (contiguous), destination block index, byte offset in that block)];
        ``block_kinds``: per destination block, ``DTYPE_F16`` / ``DTYPE_BF16`` if its fp32 sources are to be
        rounded to that type on the way (``DTYPE_F32`` or None: plain copies)."""
        assert len(items) <= MAX_COPY_SEGMENTS, f"at most {MAX_COPY_SEGMENTS} copies per plan"
        self.segs = (CopySegmentC * max(len(items), 1))()
        self.where = []
        self.keep = [src for src, _, _ in items]  # the sources stay alive as long as the plan
        for seg, (src, block, offset) in zip(self.segs, items):
            assert src.is_contiguous()
            seg.src, seg.bytes = src.data_ptr(), src.numel() * src.element_size()
            self.where.append((block, offset))
        self.n = len(items)
        self.kinds = _segment_kinds(items, block_kinds)

    def run(self, lib, device, bases) -> int:
        """``bases[i]``: address of destination block ``i``.  One launch."""
        if self.n == 0:
            return 0
        segs = self.segs
        for k, (block, offset) in enumerate(self.where):
            segs[k].dst = bases[block] + offset
        if self.kinds is not None:
            return _check(lib, lib.vmas_b200_copy_buffers_convert(segs, self.kinds, self.n, _stream(device)))
        return _check(lib, lib.vmas_b200_copy_buffers(segs, self.n, _stream(device)))


MAX_OUT_BLOCKS = 8


class EnvStepC(C.Structure):
    _fields_ = [
        ("cfg", C.c_void_p), ("tb", C.c_void_p), ("st", C.c_void_p),
        ("agents", C.c_void_p), ("n_agents", C.c_int32), ("clamp", C.c_int32),
        ("bad_flag", C.c_void_p), ("steps", C.c_void_p), ("ingest_mask", C.c_void_p),
        ("graph_exec", C.c_void_p), ("mask", C.c_void_p), ("exact_broad_phase", C.c_int32), ("fused_kernel", C.c_int32),
        ("program", C.c_void_p), ("columns", C.c_void_p), ("n_rows", C.c_int32), ("width", C.c_int32),
        ("obs_out", C.c_void_p),
        ("segs", C.c_void_p), ("seg_block", C.c_void_p), ("n_segs", C.c_int32), ("n_out_blocks", C.c_int32),
        ("out_blocks", C.c_void_p * MAX_OUT_BLOCKS),
        ("obs_block", C.c_int32), ("n_mirrors", C.c_int32), ("obs_offset", C.c_size_t),
        ("ingest_in_kernel", C.c_int32), ("obs_dtype", C.c_int32),
        ("mirror_slot", C.c_int32 * PROG_MAX_BUFFERS), ("mirror_block", C.c_int32 * PROG_MAX_BUFFERS),
        ("mirror_offset", C.c_size_t * PROG_MAX_BUFFERS),
        ("seg_kind", C.c_void_p),
    ]


class EnvStepPlan:
    """``vmas_b200_env_step`` with everything that does not change from step to step marshalled once:
    a run fills in the action tensors' addresses and the fresh output blocks, then crosses the FFI once
    (action ingest, the step itself — a captured graph or the library's own two launches — and the
    hand-out copy)."""

    def __init__(self, lib, dt: "DeviceTables", slab, agents_c, n_agents: int, clamp: bool, bad_flag, steps,
                 ingest_broad_phase: bool, graph_exec: int, copy_items, n_out_blocks: int,
                 program=None, columns=None, n_rows: int = 0, width: int = 0, obs_out=None, exact_broad_phase: int = 1,
                 obs_to=None, mirrors=(), block_kinds=None, obs_dtype: int = DTYPE_F32):
        """``obs_to``: (block, byte offset) the observation rows are written to directly (direct mode), as
        ``obs_dtype`` (``DTYPE_*``); ``mirrors``: [(program buffer slot, block, byte offset)] stores that land in
        the fresh blocks; ``block_kinds``: as ``CopyPlan`` takes them, for the hand-out copies."""
        assert len(copy_items) <= MAX_COPY_SEGMENTS and n_out_blocks <= MAX_OUT_BLOCKS and n_agents <= MAX_INGEST_AGENTS
        self.lib, self.device = lib, dt.device
        st = dt.state_struct(slab)
        segs = (CopySegmentC * max(len(copy_items), 1))()
        blocks = (C.c_int32 * max(len(copy_items), 1))()
        for k, (src, block, offset) in enumerate(copy_items):
            assert src.is_contiguous()
            segs[k].src, segs[k].dst, segs[k].bytes = src.data_ptr(), offset, src.numel() * src.element_size()
            blocks[k] = block
        c = self.c = EnvStepC()
        c.cfg, c.tb, c.st = C.addressof(dt.cfg), C.addressof(dt.tb), C.addressof(st)
        c.agents = C.addressof(agents_c) if n_agents else None
        c.n_agents, c.clamp = n_agents, int(clamp)
        c.bad_flag = None if bad_flag is None else bad_flag.data_ptr()
        c.steps = None if steps is None else steps.data_ptr()
        c.ingest_mask = dt.mask.data_ptr() if ingest_broad_phase else None
        c.graph_exec = graph_exec or None
        c.mask, c.exact_broad_phase = dt.mask.data_ptr(), exact_broad_phase
        c.program = None if program is None else C.addressof(program)
        c.columns = None if columns is None else columns.data_ptr()
        c.n_rows, c.width = n_rows, width
        c.obs_out = None if obs_out is None else obs_out.data_ptr()
        c.segs, c.seg_block = C.addressof(segs), C.addressof(blocks)
        c.n_segs, c.n_out_blocks = len(copy_items), n_out_blocks
        c.obs_block = -1
        if obs_to is not None:
            c.obs_block, c.obs_offset = obs_to
        assert len(mirrors) <= PROG_MAX_BUFFERS
        c.n_mirrors = len(mirrors)
        for k, (slot, block, offset) in enumerate(mirrors):
            c.mirror_slot[k], c.mirror_block[k], c.mirror_offset[k] = slot, block, offset
        c.obs_dtype = obs_dtype if obs_to is not None else DTYPE_F32
        kinds = _segment_kinds(copy_items, block_kinds)
        c.seg_kind = None if kinds is None else C.addressof(kinds)
        self.out_blocks = c.out_blocks
        self.agents = agents_c
        self._ref = C.addressof(c)
        self._call = lib.vmas_b200_env_step
        # everything the addresses above point into stays alive with the plan
        self.keep = (dt, slab, st, agents_c, segs, blocks, kinds, bad_flag, steps, program, columns, obs_out,
                     [src for src, _, _ in copy_items])

    def run(self) -> int:
        """(the caller has filled in ``agents[i].actions`` and ``out_blocks[j]``)"""
        return _check(self.lib, self._call(self._ref, _stream(self.device)))


def distance_shaping(lib, dt: DeviceTables, slab, pairs, factor: float, prev, dist, rew) -> int:
    """``pairs`` int32[K, 2]; ``prev`` fp32[K, B] updated in place; ``dist`` (or None) and ``rew`` fp32[K, B]."""
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_distance_shaping(
        C.byref(dt.cfg), C.byref(st), pairs.data_ptr(), int(pairs.shape[0]), float(factor), prev.data_ptr(),
        None if dist is None else dist.data_ptr(), rew.data_ptr(), _stream(dt.device),
    )
    return _check(lib, rc)


RAYS_RANGE_MINUS_DISTANCE = 1
RAYS_SPHERE_TARGETS = 2
QUERY_SPHERES = 0x100
OBS_SKIP, OBS_COPY, OBS_DIFF, OBS_REMAINDER = 0, 1, 2, 3
OBS_POS, OBS_VEL, OBS_ROT, OBS_ANG_VEL = 0, 1, 2, 3


def gather_observations(lib, dt: DeviceTables, slab, columns, n_rows: int, width: int, out, buffers=()) -> int:
    """``columns`` int32[R, F, 4] on the device, ``out`` fp32 [R, B, F]; ``buffers``: the fp32 ``[B]`` tensors
    VMAS_OBS_BUFFER columns read (see include/vmas_b200.h)."""
    st = dt.state_struct(slab)
    if buffers:
        ptrs = (C.c_void_p * len(buffers))(*[b.data_ptr() for b in buffers])
        rc = lib.vmas_b200_gather_observations_buffers(
            C.byref(dt.cfg), C.byref(st), columns.data_ptr(), int(n_rows), int(width), out.data_ptr(), ptrs,
            len(buffers), _stream(dt.device),
        )
        return _check(lib, rc)
    rc = lib.vmas_b200_gather_observations(
        C.byref(dt.cfg), C.byref(st), columns.data_ptr(), int(n_rows), int(width), out.data_ptr(), _stream(dt.device)
    )
    return _check(lib, rc)


def pair_query_batched(lib, dt: DeviceTables, slab, pairs, mode: int, out) -> int:
    st = dt.state_struct(slab)
    rc = lib.vmas_b200_pair_query_batched(
        C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), pairs.data_ptr(), int(pairs.shape[0]), mode, out.data_ptr(),
        _stream(dt.device),
    )
    return _check(lib, rc)


class SlabHandle:
    """What the reset entry points need of a world: its sizes and the slab's device pointers.  Unlike
    :class:`DeviceTables` it does not need the compiled plan, so a world can be reset before its
    collision structure is final (scenario collision filters may read state the first reset creates)."""

    def __init__(self, slab):
        for t in slab.tensors():
            assert t.is_contiguous() and t.dtype == torch.float32 and t.device.type == "cuda"
        self.device = slab.pos.device
        self.cfg = WorldConfig()
        self.cfg.batch_dim = slab.batch_dim
        self.cfg.n_entities = slab.n_entities
        self.cfg.n_agents = slab.n_agents
        self.st = StateC()
        self.st.pos, self.st.vel, self.st.rot, self.st.ang_vel, self.st.force, self.st.torque = (
            t.data_ptr() for t in slab.tensors()
        )


def reset_state(lib, handle: SlabHandle, env_index, env_mask, reset_count) -> int:
    """Zero the state rows of the selected envs (``env_index`` int or None, ``env_mask`` uint8
    ``[B]`` or None) and bump their episode counters (``reset_count`` int32 ``[B]`` or None)."""
    rc = lib.vmas_b200_reset_state(
        C.byref(handle.cfg), C.byref(handle.st), -1 if env_index is None else int(env_index),
        None if env_mask is None else env_mask.data_ptr(),
        None if reset_count is None else reset_count.data_ptr(), _stream(handle.device),
    )
    return _check(lib, rc)


def spawn_entities(lib, handle: SlabHandle, spawn: SpawnC) -> int:
    """``spawn``: a filled ``SpawnC`` (device pointers as integers)."""
    rc = lib.vmas_b200_spawn_entities(C.byref(handle.cfg), C.byref(handle.st), C.byref(spawn), _stream(handle.device))
    return _check(lib, rc)
