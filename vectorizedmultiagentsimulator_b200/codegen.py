"""Generates ``csrc/generated/specializations.cuh``: constexpr world tables for the specialised kernel.

``csrc/spec_kernel.cuh`` is a hand-written template that turns a compile-time world description
into a fully unrolled, register-resident substep kernel.  This module only emits the *data* it
is instantiated with — one ``struct World_<hash>`` per preset world (the BASELINE.json configs
and the shipped scenarios' defaults) — plus the registry the C ABI looks specialisations up in
by a 64-bit hash of the world description.  Worlds without a specialisation run on the generic
table-driven kernels; both produce identical bits (tests/test_cabi_gpu.py).

    python -m vectorizedmultiagentsimulator_b200.codegen        # rewrite the generated header
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Tuple

import numpy as np

from . import _native as N
from .simulator import plan as P

HERE = os.path.dirname(os.path.abspath(__file__))
GENERATED = os.path.join(HERE, "csrc", "generated", "specializations.cuh")

#: worlds that get an ahead-of-time specialisation: (scenario, kwargs[, tuning]).
#: tuning["min_blocks"]: resident blocks per SM the register allocator leaves room for (default: the
#: build's SPEC_MIN_BLOCKS = 8, i.e. <= 128 registers at 64 threads per block).  Chosen per world by
#: measurement: stock transport with 12 (80 registers, 24 warps / SM), the others at the default (not yet
#: re-measured on H100, which has the same 64 K registers per SM).
PRESETS: List[Tuple] = [
    ("balance", dict(n_agents=4)),  # BASELINE.json configs[0], [1]
    ("balance", dict()),
    ("transport", dict(n_agents=4), dict(min_blocks=12)),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3)),  # BASELINE.json configs[2] variant
    ("navigation", dict(n_agents=8)),  # configs[3]
    ("navigation", dict()),
    ("flocking", dict(n_agents=5)),  # configs[4]
    ("flocking", dict()),
]

#: specialisation is skipped for worlds whose unrolled code would be unreasonably large
MAX_ENTITIES = 24
MAX_ITEM_COST = 400  # in units of one segment/segment test


def world_hash(desc: P.WorldDescription) -> int:
    """FNV-1a 64 of everything that shapes the kernel (not the batch size, not entity names)."""
    d = json.loads(desc.to_json())
    d.pop("batch_dim")
    for e in d["entities"]:
        e.pop("name")
        for flag in ("gravity_per_env", "mass_per_env", "lin_fric_per_env", "ang_fric_per_env"):
            if not e.get(flag):
                e.pop(flag, None)  # absent in descriptions written before the field existed
    blob = json.dumps(d, sort_keys=True).encode()
    h = 0xCBF29CE484222325
    for byte in blob:
        h ^= byte
        h = (h * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def _item_cost(kind: int) -> int:
    return {P.K_JOINT: 1, P.K_SS: 1, P.K_LS: 1, P.K_LL: 1, P.K_BS: 1, P.K_BL: 4, P.K_BB: 32}[kind]


def specializable(desc: P.WorldDescription, per_env: bool = False) -> bool:
    """Whether ``desc`` gets the specialised kernels.  ``per_env``: worlds with per-env masses, friction
    coefficients or gravity qualify too (their step_spec_kernel reads SpecArgs.ent_params / ent_gravity; they
    get neither the tile kernel nor a whole-step kernel), else they do not."""
    if desc.n_entities > MAX_ENTITIES or desc.n_entities == 0:
        return False
    if not per_env and has_per_env_params(desc):
        return False
    return sum(_item_cost(it["kind"]) for it in desc.items) <= MAX_ITEM_COST


def has_per_env_params(desc: P.WorldDescription) -> bool:
    """Some entity's mass, friction coefficient or gravity is given per env."""
    flags = ("gravity_per_env", "mass_per_env", "lin_fric_per_env", "ang_fric_per_env")
    return any(e.get(f) for e in desc.entities for f in flags)


def _f(x) -> str:
    v = float(np.float32(x))
    if v != v or v in (float("inf"), float("-inf")):
        raise ValueError(f"non-finite constant {x} in world description")
    s = f"{v:.9g}"
    if "e" not in s and "." not in s:
        s += ".0"
    return s + "f"


def emit_world(desc: P.WorldDescription, label: str, tuning: Dict = None) -> Tuple[str, str, int]:
    """C++ text of one world struct.  Returns (struct name, text, hash)."""
    min_blocks = (tuning or {}).get("min_blocks", "SPEC_MIN_BLOCKS")
    tables = P.build_tables(desc)
    h = world_hash(desc)
    # the entities' per-env attributes (spec_kernel.cuh reads them from SpecArgs behind `if constexpr`);
    # emitted only when there are any, so that every other world's text stays as it was
    env_mask = [int(f) & (P.F_GRAVITY_ENV | P.F_PARAMS_ENV) for f in tables.ent_i32[: desc.n_entities, 1]]
    per_env = any(env_mask)
    name = f"World_{h:016x}"
    E, NI = desc.n_entities, len(desc.items)
    ef, ei = tables.ent_f32, tables.ent_i32
    lines = [f"// {label}: E={E} items={NI} substeps={desc.substeps}", f"struct {name} {{"]
    lines.append(f"  static constexpr int E = {E}, A = {desc.n_agents}, NI = {NI}, N_JOINTS = {tables.n_joints};")
    lines.append(
        f"  static constexpr int MASK_WORDS = {(tables.n_masked + 31) // 32}, BLOCK = SPEC_BLOCK, "
        f"MIN_BLOCKS = {min_blocks};"
    )
    d = desc
    lines.append(
        "  static constexpr CfgC cfg = {"
        f"{d.substeps}, {int(d.x_semidim is not None)}, {int(d.y_semidim is not None)}, "
        f"{int(any(g != 0.0 for g in d.gravity))}, {_f(d.dt / d.substeps)}, {_f(d.x_semidim or 0.0)}, "
        f"{_f(d.y_semidim or 0.0)}, {_f(d.collision_force)}, {_f(d.joint_force)}, "
        f"{_f(d.torque_constraint_force)}, {_f(d.contact_margin)}, {_f(d.gravity[0])}, {_f(d.gravity[1])}}};"
    )
    lines.append(f"  static constexpr EntC ent[{max(E, 1)}] = {{")
    for e in range(E):
        r = ef[e]
        cols = [
            P.EF_D0, P.EF_D1, P.EF_MASS, P.EF_INERTIA, P.EF_DRAG_MULT, P.EF_LIN_FRIC, P.EF_ANG_FRIC, P.EF_GRAV_X,
            P.EF_GRAV_Y, P.EF_MAX_SPEED, P.EF_V_RANGE, P.EF_MAX_F, P.EF_F_RANGE, P.EF_MAX_T, P.EF_T_RANGE,
            P.EF_CIRC_R, P.EF_R_PLUS_LMD,
        ] + ([P.EF_INERTIA_K0, P.EF_INERTIA_K1] if per_env else [])
        vals = ", ".join(_f(r[c]) for c in cols)
        lines.append(f"      {{{int(ei[e, 0])}, {int(ei[e, 1])}, {int(ei[e, 2])}, {vals}}},  // {desc.entities[e]['name']}")
    lines.append("  };")
    if per_env:
        lines.append(f"  static constexpr int PER_ENV[{E}] = {{{', '.join(str(m) for m in env_mask)}}};")
    lines.append(f"  static constexpr ItemC item[{max(NI, 1)}] = {{")
    if NI == 0:
        lines.append("      {0, 0, 0, 0, -1, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f},")
    for k in range(NI):
        ii, f32 = tables.item_i32[k], tables.item_f32[k]
        flags = int(ii[3]) & 0xFF
        vals = ", ".join(
            _f(f32[c]) for c in (P.IF_DMIN_BASE, P.IF_AX, P.IF_AY, P.IF_BX, P.IF_BY, P.IF_DIST, P.IF_FIXED_ROT, P.IF_BROAD_THR)
        )
        lines.append(
            f"      {{{int(ii[0])}, {int(ii[1])}, {int(ii[2])}, {flags}, {int(tables.mask_slot[k])}, {vals}}},"
            f"  // {P.KIND_NAMES[int(ii[0])]}"
        )
    lines.append("  };")
    lines.append("};")
    return name, "\n".join(lines), h


# ---- the action prologue of the one-kernel step -------------------------------------------------------------------
#: the action models the prologue runs (``VMAS_DYN_*``: holonomic, holonomic with rotation, forward, rotation,
#: differential drive) and the action size each takes: the model's own.  Left to the ingest launch: the kinematic
#: bicycle (its prologue measured slower than its two-launch step on the H100, DESIGN §7.4) and the drone (a 12-state
#: RK4 per agent).
PROLOGUE_MODELS = {N.DYN_HOLONOMIC: 2, N.DYN_HOLONOMIC_ROT: 3, N.DYN_FORWARD: 1, N.DYN_ROTATION: 1,
                   N.DYN_DIFF_DRIVE: 2}


def dynamics_code(dynamics):
    """``VMAS_DYN_*`` of an agent's dynamics model (exact types: a subclass may override ``process_action``), or
    None if the ingest kernel does not implement it."""
    from .simulator.dynamics.basic import Forward, Holonomic, HolonomicWithRotation, Rotation, Static
    from .simulator.dynamics.diff_drive import DiffDrive
    from .simulator.dynamics.drone import Drone
    from .simulator.dynamics.kinematic_bicycle import KinematicBicycle

    return {
        Holonomic: N.DYN_HOLONOMIC, HolonomicWithRotation: N.DYN_HOLONOMIC_ROT, Forward: N.DYN_FORWARD,
        Rotation: N.DYN_ROTATION, Static: N.DYN_NONE, DiffDrive: N.DYN_DIFF_DRIVE, KinematicBicycle: N.DYN_BICYCLE,
        Drone: N.DYN_DRONE,
    }.get(type(dynamics))


def dynamics_params(agent, dyn: int) -> List[float]:
    """``VmasAgentActions::dyn_params`` of a kinematic model: dt, mass, moment of inertia, rk4 (1 / 0), then the
    bicycle's l_f, l_r, max steering angle or the drone's I_xx, I_yy, I_zz, g.  Zeros for the other models."""
    params = [0.0] * 8
    if dyn >= N.DYN_DIFF_DRIVE:
        model = agent.dynamics
        params[:4] = [float(model.dt), float(agent.mass), float(agent.moment_of_inertia),
                      1.0 if model.integration == "rk4" else 0.0]
        if dyn == N.DYN_BICYCLE:
            params[4:7] = [float(model.l_f), float(model.l_r), float(model.max_steering_angle)]
        elif dyn == N.DYN_DRONE:
            params[4:8] = [float(model.I_xx), float(model.I_yy), float(model.I_zz), float(model.g)]
    return params


def prologue_acts(agents, kind: int = N.ACT_CONTINUOUS) -> tuple:
    """The ``acts`` of a whole-step kernel whose prologue ingests the actions of ``agents`` (the policy agents with
    action components, in ingest order; each with the fields of ``VmasAgentActions``: ``agent_index``,
    ``dynamics``, ``action_size``, ``u_range``, ``u_multiplier``, ``nvec``, ``dyn_params``), or ``()`` if the
    prologue does not take them all: every agent's model must be in ``PROLOGUE_MODELS`` with its own action size,
    and there are at most ``VMAS_MAX_INGEST_AGENTS``.  ``kind``: ``VMAS_ACT_*`` of the action space.

    An entry is ``(agent row, u_range x 2, u_multiplier x 2)`` for a holonomic agent with 2 components and continuous
    actions, plus ``(kind, nvec x 2)`` for discrete ones: the text and the key of those kernels stay what they were
    before the other models.  Other agents: ``(row, u_range x 2, u_multiplier x 2, kind, nvec x 2, dynamics, size,
    u_range[2:4], u_multiplier[2:4], nvec[2:4], dyn_params x 8)`` (``ActC`` in csrc/spec_kernel.cuh)."""
    if not agents or len(agents) > N.MAX_INGEST_AGENTS:
        return ()
    acts = []
    for c in agents:
        dyn, size = int(c.dynamics), int(c.action_size)
        if PROLOGUE_MODELS.get(dyn) != size:
            return ()
        rng = [float(c.u_range[j]) if j < size else 0.0 for j in range(4)]
        mul = [float(c.u_multiplier[j]) if j < size else 0.0 for j in range(4)]
        nvec = [int(c.nvec[j]) if kind != N.ACT_CONTINUOUS and j < size else 0 for j in range(4)]
        act = (int(c.agent_index), rng[0], rng[1], mul[0], mul[1])
        if dyn == N.DYN_HOLONOMIC and size == 2:
            acts.append(act + (() if kind == N.ACT_CONTINUOUS else (int(kind), nvec[0], nvec[1])))
        else:
            acts.append(act + (int(kind), nvec[0], nvec[1], dyn, size, rng[2], rng[3], mul[2], mul[3], nvec[2],
                               nvec[3]) + tuple(float(c.dyn_params[j]) for j in range(8)))
    return tuple(acts)


def _act_fields(act) -> list:
    """One ``acts`` entry as the typed list the key hashes (see ``prologue_acts``)."""
    fields = [int(act[0])] + [_f(v) for v in act[1:5]] + [int(v) for v in act[5:10]]
    if len(act) > 10:
        fields += [_f(v) for v in act[10:14]] + [int(v) for v in act[14:16]] + [_f(v) for v in act[16:]]
    return fields


# ---- the LIDAR stage of the whole-step kernel's epilogue ------------------------------------------------------------
#: the most targets one LIDAR of a whole-step kernel casts its rays at (``SPEC_LIDAR_MAX_TARGETS`` in
#: csrc/spec_kernel.cuh: the epilogue unrolls every ray against every target).  A plan with a sensor that sees more
#: stays on the captured graph, which casts them with ``cast_rays_batched_kernel``.
MAX_LIDAR_TARGETS = 16


def lidar_sensors(lidars, index_of, ray_targets):
    """The LIDAR table of a whole-step kernel: ``(sensors, flip)`` for the ``lidars`` of ``ObservationPlan.compile``
    (``[(row, first column, sensor, range_minus_distance)]``), or None if a sensor sees more than
    ``MAX_LIDAR_TARGETS`` targets.  A sensor is ``(source entity, targets, angles, max_range, row, first column)``:
    the targets in ``ray_targets`` order, the angles and the range as the fp32 values ``cast_rays_batched_kernel``
    reads.  ``flip``: the readings are stored as ``max_range - distance`` (one setting per plan, as
    ``backend.observe`` takes it)."""
    sensors = []
    for row, col, s, _ in lidars:
        targets = tuple(int(t) for t in ray_targets(s.agent, s.entity_filter))
        if len(targets) > MAX_LIDAR_TARGETS:
            return None
        angles = tuple(float(x) for x in np.asarray(s._angles[0].detach().cpu(), dtype=np.float32))
        sensors.append((int(index_of(s.agent)), targets, angles, float(np.float32(s._max_range)), int(row), int(col)))
    return tuple(sensors), bool(lidars[0][3]) if lidars else False


def post_hash(cols, instrs, acts=(), obs_dtype: int = 0, lidar=None) -> int:
    """FNV-1a 64 of what a whole-step kernel does around the substeps: the observation plan's column table
    (int32 ``[rows, width, 4]`` or None), the step program's instructions ``[(op, dst, a, b, arg, imm)]`` with
    entity indices resolved, the action ingest of the policy agents (``prologue_acts``; empty: actions are ingested
    by a launch of their own), the type of the observation rows (``VMAS_DTYPE_*``; fp32 adds nothing to the
    hash) and the LIDAR table (``lidar_sensors``; None or no sensor adds nothing)."""
    parts = [None if cols is None else [list(cols.shape), [int(x) for x in cols.reshape(-1)]],
             [[int(op), int(dst), int(a), int(b), int(arg), _f(imm)] for op, dst, a, b, arg, imm in instrs],
             [_act_fields(act) for act in acts]]
    if obs_dtype:
        parts.append(int(obs_dtype))
    if lidar and lidar[0]:
        sensors, flip = lidar
        parts.append([int(flip), [[src, list(targets), [_f(a) for a in angles], _f(rng), row, col]
                                  for src, targets, angles, rng, row, col in sensors]])
    blob = json.dumps(parts).encode()
    h = 0xCBF29CE484222325
    for byte in blob:
        h ^= byte
        h = (h * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def fuse_value_columns(cols, buffer_sources, instrs):
    """The column table of an observation plan for a whole-step kernel: value columns (``observe.value`` of a
    program output; OP_BUFFER = 4, index into ``buffer_sources``) become reads of the program register that
    output stores (OP_REG = 5) — program and observation rows run in one thread there."""
    OP_BUFFER, OP_REG, STORES = 4, 5, (20, 21)
    if cols is None or not buffer_sources:
        return cols
    reg_of = {b: a for op, _, a, b, _, _ in instrs if op in STORES}
    cols = cols.copy()
    for row in cols.reshape(-1, 4):
        if row[0] == OP_BUFFER:
            row[0], row[1] = OP_REG, reg_of[buffer_sources[int(row[1])]._slot]
    return cols


def emit_post(cols, instrs, acts=(), obs_dtype: int = 0, lidar=None) -> Tuple[str, str, int]:
    """C++ text of one epilogue (+ ingest prologue) struct (``spec_epilogue`` / ``spec_ingest`` / ``spec_lidar`` in
    csrc/spec_kernel.cuh).  ``obs_dtype``: what the observation rows are stored as (``VMAS_DTYPE_F32`` = 0,
    ``VMAS_DTYPE_F16`` = 1, ``VMAS_DTYPE_BF16`` = 2).  ``lidar``: ``lidar_sensors`` of the plan's LIDAR terms (their
    columns are SKIP in ``cols``).  Returns (name, text, hash)."""
    h = post_hash(cols, instrs, acts, obs_dtype, lidar)
    name = f"Post_{h:016x}"
    rows, width = (0, 0) if cols is None else (int(cols.shape[0]), int(cols.shape[1]))
    lines = [f"struct {name} {{"]
    lines.append(
        f"  static constexpr int N_PROG = {len(instrs)}, OBS_ROWS = {rows}, OBS_WIDTH = {width}, N_ACT = {len(acts)}, "
        f"OBS_DTYPE = {int(obs_dtype)};"
    )
    lines.append(f"  static constexpr ActC act[{max(len(acts), 1)}] = {{")
    for act in acts:
        agent, r0, r1, m0, m1 = act[:5]
        tail = "".join(f", {int(v)}" for v in act[5:10])  # (kind, n0, n1[, dyn, size]: else the defaults)
        if len(act) > 10:
            tail += "".join(f", {_f(v)}" for v in act[10:14]) + "".join(f", {int(v)}" for v in act[14:16])
            tail += ", {" + ", ".join(_f(v) for v in act[16:]) + "}"
        lines.append(f"      {{{int(agent)}, {_f(r0)}, {_f(r1)}, {_f(m0)}, {_f(m1)}{tail}}},")
    if not acts:
        lines.append("      {0, 0.f, 0.f, 0.f, 0.f},")
    lines.append("  };")
    lines.append(f"  static constexpr ProgC prog[{max(len(instrs), 1)}] = {{")
    for op, dst, a, b, arg, imm in instrs:
        lines.append(f"      {{{int(op)}, {int(dst)}, {int(a)}, {int(b)}, {int(arg)}, {_f(imm)}}},")
    if not instrs:
        lines.append("      {0, 0, 0, 0, 0, 0.f},")
    lines.append("  };")
    lines.append(f"  static constexpr ObsColC obs[{max(rows * width, 1)}] = {{")
    if rows * width == 0:
        lines.append("      {0, 0, 0, 0.f},")
    else:
        flat = cols.reshape(-1, 4)
        for op, src, src2, par in flat:
            par_f = float(np.array([par], dtype=np.int32).view(np.float32)[0])
            lines.append(f"      {{{int(op)}, {int(src)}, {int(src2)}, {_f(par_f)}}},")
    lines.append("  };")
    if lidar and lidar[0]:  # (members a plan without LIDAR terms does not have: its text stays as it was)
        sensors, flip = lidar
        n_rays = {len(angles) for _, _, angles, _, _, _ in sensors}
        if len(n_rays) != 1:
            raise ValueError("LIDARs of one observation plan must have the same number of rays")
        R = n_rays.pop()
        lines.append(f"  static constexpr int N_LIDAR = {len(sensors)}, LIDAR_RAYS = {R}, LIDAR_FLIP = {int(flip)};")
        lines.append(f"  static constexpr LidarC lidar[{len(sensors)}] = {{")
        for src, targets, angles, rng, row, col in sensors:
            if len(targets) > MAX_LIDAR_TARGETS:
                raise ValueError(f"a LIDAR of a whole-step kernel sees at most {MAX_LIDAR_TARGETS} targets")
            lines.append(f"      {{{src}, {row}, {col}, {_f(rng)}, {len(targets)}, {{{', '.join(str(t) for t in targets)}}}}},")
        lines.append("  };")
        lines.append(f"  static constexpr float lidar_angle[{len(sensors) * R}] = {{")
        for _, _, angles, _, _, _ in sensors:
            lines.append("      " + ", ".join(_f(a) for a in angles) + ",")
        lines.append("  };")
    lines.append("};")
    return name, "\n".join(lines), h


def preset_descriptions() -> List[Tuple[str, P.WorldDescription, Dict]]:
    """Builds every preset world on the CPU (construction only, no physics) and describes it."""
    import torch

    from . import scenarios

    out = []
    for scenario, kwargs, *tuning in PRESETS:
        sc = scenarios.load(scenario + ".py").Scenario()
        world = sc.env_make_world(1, torch.device("cpu"), **dict(kwargs))
        label = scenario + "(" + ", ".join(f"{k}={v}" for k, v in kwargs.items()) + ")"
        out.append((label, P.describe_world(world), tuning[0] if tuning else None))
    return out


def generate(path: str = GENERATED) -> List[Tuple[str, int]]:
    worlds, seen = [], set()
    for label, desc, tuning in preset_descriptions():
        if not specializable(desc):
            continue
        name, text, h = emit_world(desc, label, tuning)
        if h in seen:
            continue
        seen.add(h)
        worlds.append((label, name, text, h, desc))
    parts = [
        "// GENERATED by vectorizedmultiagentsimulator_b200/codegen.py — do not edit.",
        "// constexpr world tables the specialised substep kernel (spec_kernel.cuh) is instantiated with.",
        "#pragma once",
        '#include "../spec_kernel.cuh"',
        '#include "../spec_tile_kernel.cuh"',
        "",
        "namespace vmas {",
        "",
    ]
    for _, _, text, _, _ in worlds:
        parts += [text, ""]
    parts.append("#ifdef __CUDACC__")
    parts.append("static const SpecEntry kSpecs[] = {")
    for label, name, _, h, desc in worlds:
        parts.append(
            f'    {{0x{h:016x}ull, "{label}", {desc.n_entities}, {len(desc.items)}, &launch_spec<{name}>, '
            f"&launch_tile<{name}>, TileLayout<{name}>::SUPPORTED}},"
        )
    if not worlds:
        parts.append('    {0ull, "", 0, 0, nullptr, nullptr, false},')
    parts.append("};")
    parts.append(f"static const int kNumSpecs = {len(worlds)};")
    parts.append("#endif")
    # the same worlds as a type list, for code that instantiates a template per world (tests/hostsim)
    parts.append("#define VMAS_FOR_EACH_SPEC_WORLD(X) \\")
    parts.append(" \\\n".join(f"  X({i}, {name}, 0x{h:016x}ull)" for i, (_, name, _, h, _) in enumerate(worlds)))
    parts += ["", "}  // namespace vmas", ""]
    text = "\n".join(parts)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if not os.path.exists(path) or open(path).read() != text:
        with open(path, "w") as fh:
            fh.write(text)
    return [(label, h) for label, _, _, h, _ in worlds]


if __name__ == "__main__":
    for label, h in generate():
        print(f"{h:016x}  {label}")
