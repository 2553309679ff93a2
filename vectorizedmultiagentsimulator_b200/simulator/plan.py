"""Plan compiler: flattens a world's static structure into the tables the kernels read.

``describe_world`` walks a world through its *public* attributes only (entities, shapes,
flags, joints), so it works both on this package's :class:`~.core.World` and — in the parity
tests — on a world built by the unmodified reference.  The result is a plain, JSON-able
:class:`WorldDescription`; ``build_tables`` turns it into the numpy tables uploaded to the
GPU (and consumed, unchanged, by the CPU oracle under ``oracle/``).

What is evaluated here, once, instead of every substep as the reference does:

* the static predicates of ``World.collides`` (ref core.py:2788-2796) incl. the user's
  ``collision_filter`` callables, and the joint lookup (ref core.py:2112-2174);
* the bucket order joints, S-S, L-S, L-L, B-S, B-L, B-B (ref core.py:2175-2189), which fixes
  the order forces are accumulated in;
* every fp32 rounding the reference applies to python scalars before they meet a tensor
  (SURVEY.md Appendix A, "threshold rounding").
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from .utils import LINE_MIN_DIST

# shape kinds
SHAPE_SPHERE, SHAPE_BOX, SHAPE_LINE = 0, 1, 2
# work-item kinds, in accumulation order
K_JOINT, K_SS, K_LS, K_LL, K_BS, K_BL, K_BB = 0, 1, 2, 3, 4, 5, 6
KIND_NAMES = ["joint", "sphere-sphere", "line-sphere", "line-line", "box-sphere", "box-line", "box-box"]

# entity flag bits (ent_i32[:, 1])
F_MOVABLE = 1 << 0
F_ROTATABLE = 1 << 1
F_HOLLOW = 1 << 2
F_AGENT = 1 << 3
F_LIN_FRIC = 1 << 4
F_ANG_FRIC = 1 << 5
F_GRAVITY = 1 << 6
F_MAX_SPEED = 1 << 7
F_V_RANGE = 1 << 8
F_MAX_F = 1 << 9
F_F_RANGE = 1 << 10
F_MAX_T = 1 << 11
F_T_RANGE = 1 << 12
F_TRIG = 1 << 13  # kernel must evaluate sin/cos of this entity's rotation
F_GRAVITY_ENV = 1 << 14  # per-env gravity rows in ent_gravity[B, E, 2]
F_MASS_ENV = 1 << 15  # per-env mass in ent_params[B, E, 4] column 0 (moment of inertia derived in the kernel)
F_LIN_FRIC_ENV = 1 << 16  # per-env linear-friction coefficient, ent_params column 1
F_ANG_FRIC_ENV = 1 << 17  # per-env angular-friction coefficient, ent_params column 2
F_PARAMS_ENV = F_MASS_ENV | F_LIN_FRIC_ENV | F_ANG_FRIC_ENV

# columns of ent_f32
(
    EF_D0,
    EF_D1,
    EF_MASS,
    EF_INERTIA,
    EF_DRAG_MULT,
    EF_LIN_FRIC,
    EF_ANG_FRIC,
    EF_GRAV_X,
    EF_GRAV_Y,
    EF_MAX_SPEED,
    EF_V_RANGE,
    EF_MAX_F,
    EF_F_RANGE,
    EF_MAX_T,
    EF_T_RANGE,
    EF_CIRC_R,
    EF_R_PLUS_LMD,
    EF_INERTIA_K0,
    EF_INERTIA_K1,
) = range(19)
EF_COLS = 20
#: columns of the per-env parameter table ent_params[B, E, EP_COLS]
EP_MASS, EP_LIN_FRIC, EP_ANG_FRIC = 0, 1, 2
EP_COLS = 4
#: what a per-env attribute's scalar field holds in a description: the hash does not see the values
PER_ENV_PLACEHOLDER = 1.0
EI_COLS = 4  # shape kind, flags, agent index, reserved

# columns of item_f32 / item_i32
(IF_BROAD_THR, IF_DMIN_BASE, IF_AX, IF_AY, IF_BX, IF_BY, IF_DIST, IF_FIXED_ROT) = range(8)
IF_COLS = 8
II_COLS = 4  # kind, a, b, flags
IFLAG_JOINT_ROTATE = 1
IFLAG_JOINT_ROT_PER_ENV = 2
IFLAG_ALWAYS_ACTIVE = 4  # broad phase not applied (joints)


def _shape_kind(shape) -> int:
    name = type(shape).__name__
    if name == "Sphere":
        return SHAPE_SPHERE
    if name == "Box":
        return SHAPE_BOX
    if name == "Line":
        return SHAPE_LINE
    raise RuntimeError(f"Shape {shape} is not supported by the CUDA physics kernels")


def _is_agent(entity) -> bool:
    return hasattr(entity, "action") and hasattr(entity, "dynamics")


#: action models that back-solve the force / torque from the agent's mass in the action ingest
KINEMATIC_DYNAMICS = ("DiffDrive", "KinematicBicycle", "Drone")


def _is_per_env(entity, attr) -> bool:
    """True if ``entity.<attr>`` is a ``[batch_dim, 1]`` tensor (mass, linear / angular friction)."""
    v = getattr(entity, attr, None)
    if v is None or isinstance(v, (int, float)):
        return False
    if hasattr(v, "dim") and v.dim() == 0:
        return False
    if hasattr(v, "shape") and v.dim() == 2 and v.shape[1] == 1:
        return True
    raise NotImplementedError(
        f"Entity '{entity.name}': {attr} must be a python number or a [batch_dim, 1] tensor, got shape "
        f"{tuple(getattr(v, 'shape', ()))}"
    )


def inertia_constants(shape_kind: int, d0: float, d1: float):
    """(K0, K1) with moment_of_inertia(m) = fl(fl(K0 * m) * K1) for a per-env fp32 mass ``m``: the
    python-double factors of ref core.py:123-124, 160-161, 187-188, each rounded once to fp32."""
    if shape_kind == SHAPE_SPHERE:
        return 1 / 2, d0**2
    if shape_kind == SHAPE_BOX:
        return 1 / 12, d0**2 + d1**2
    return 1 / 12, d0**2


def _as_pair(value):
    """Entity/world gravity as an (x, y) pair of python floats, or None for per-env tensors."""
    if value is None:
        return None
    arr = np.asarray(value.detach().cpu().numpy() if hasattr(value, "detach") else value, dtype=np.float32)
    if arr.ndim == 0:
        return (float(arr), float(arr))
    if arr.ndim == 1 and arr.shape[0] == 2:
        return (float(arr[0]), float(arr[1]))
    return None


@dataclass
class WorldDescription:
    batch_dim: int
    substeps: int
    dt: float
    drag: float
    linear_friction: float
    angular_friction: float
    x_semidim: Optional[float]
    y_semidim: Optional[float]
    collision_force: float
    joint_force: float
    torque_constraint_force: float
    contact_margin: float
    gravity: List[float]
    entities: List[Dict] = field(default_factory=list)
    items: List[Dict] = field(default_factory=list)

    @property
    def n_entities(self):
        return len(self.entities)

    @property
    def n_agents(self):
        return sum(1 for e in self.entities if e["is_agent"])

    @property
    def n_joints(self):
        return sum(1 for it in self.items if it["kind"] == K_JOINT)

    def to_json(self) -> str:
        return json.dumps(self.__dict__)

    @staticmethod
    def from_json(text: str) -> "WorldDescription":
        return WorldDescription(**json.loads(text))


def describe_entity(entity, agent_index: int) -> Dict:
    shape = entity.shape
    kind = _shape_kind(shape)
    if kind == SHAPE_SPHERE:
        d0, d1, hollow = shape.radius, 0.0, False
    elif kind == SHAPE_BOX:
        d0, d1, hollow = shape.length, shape.width, bool(shape.hollow)
    else:
        d0, d1, hollow = shape.length, 0.0, False
    is_agent = _is_agent(entity)
    gravity = getattr(entity, "gravity", None)
    gravity_pair = _as_pair(gravity)
    gravity_per_env = gravity is not None and gravity_pair is None
    if gravity_per_env and not (hasattr(gravity, "shape") and tuple(gravity.shape[-1:]) == (2,) and gravity.dim() == 2):
        raise NotImplementedError(
            f"Entity '{entity.name}': gravity must be a scalar, an (x, y) pair or a [batch_dim, 2] tensor"
        )
    per_env = {attr: _is_per_env(entity, attr) for attr in ("mass", "linear_friction", "angular_friction")}
    if per_env["mass"] and type(getattr(entity, "dynamics", None)).__name__ in KINEMATIC_DYNAMICS:
        raise NotImplementedError(
            f"Entity '{entity.name}': a per-env mass on an agent whose action model reads the mass "
            f"({type(entity.dynamics).__name__}) is out of scope; give it a scalar mass"
        )

    def scalar(attr):
        v = getattr(entity, attr, None)
        return None if v is None else (PER_ENV_PLACEHOLDER if per_env[attr] else float(v))

    def opt(name):
        v = getattr(entity, name, None) if (is_agent or name in ("v_range", "max_speed")) else None
        return None if v is None else float(v)

    return dict(
        name=entity.name,
        is_agent=is_agent,
        agent_index=agent_index if is_agent else -1,
        shape=kind,
        d0=float(d0),
        d1=float(d1),
        hollow=hollow,
        movable=bool(entity.movable),
        rotatable=bool(entity.rotatable),
        mass=scalar("mass"),
        inertia=PER_ENV_PLACEHOLDER if per_env["mass"] else float(entity.moment_of_inertia),
        drag=None if entity.drag is None else float(entity.drag),
        linear_friction=scalar("linear_friction"),
        angular_friction=scalar("angular_friction"),
        gravity=None if gravity_pair is None else list(gravity_pair),
        gravity_per_env=bool(gravity_per_env),
        mass_per_env=per_env["mass"],
        lin_fric_per_env=per_env["linear_friction"],
        ang_fric_per_env=per_env["angular_friction"],
        max_speed=opt("max_speed"),
        v_range=opt("v_range"),
        max_f=opt("max_f"),
        f_range=opt("f_range"),
        max_t=opt("max_t"),
        t_range=opt("t_range"),
        circ_radius=float(shape.circumscribed_radius()),
    )


def _static_collides(world, a, b) -> bool:
    if (not a.collides(b)) or (not b.collides(a)) or a is b:
        return False
    if not a.movable and not a.rotatable and not b.movable and not b.rotatable:
        return False
    return True


def describe_world(world) -> WorldDescription:
    """Flatten ``world`` (this package's or the reference's) into a :class:`WorldDescription`."""
    entities = list(world.entities)
    agents = list(world.agents)
    index_of = {id(e): i for i, e in enumerate(entities)}
    agent_index = {id(a): j for j, a in enumerate(agents)}

    gravity = _as_pair(world._gravity)
    desc = WorldDescription(
        batch_dim=int(world.batch_dim),
        substeps=int(world._substeps),
        dt=float(world._dt),
        drag=float(world._drag),
        linear_friction=float(world._linear_friction),
        angular_friction=float(world._angular_friction),
        x_semidim=None if world._x_semidim is None else float(world._x_semidim),
        y_semidim=None if world._y_semidim is None else float(world._y_semidim),
        collision_force=float(world._collision_force),
        joint_force=float(world._joint_force),
        torque_constraint_force=float(world._torque_constraint_force),
        contact_margin=float(world._contact_margin),
        gravity=[gravity[0], gravity[1]],
    )
    for e in entities:
        desc.entities.append(describe_entity(e, agent_index.get(id(e), -1)))

    joints_by_names = dict(world._joints)
    joint_items: List[Dict] = []
    buckets: Dict[int, List[Dict]] = {k: [] for k in (K_SS, K_LS, K_LL, K_BS, K_BL, K_BB)}
    for ia, ea in enumerate(entities):
        for ib in range(ia + 1, len(entities)):
            eb = entities[ib]
            constraint = joints_by_names.get(frozenset({ea.name, eb.name}))
            if constraint is not None:
                ca, cb = constraint.entity_a, constraint.entity_b
                fixed = constraint.fixed_rotation
                per_env = not isinstance(fixed, (int, float))
                delta_a = ca.shape.get_delta_from_anchor(constraint.anchor_a)
                delta_b = cb.shape.get_delta_from_anchor(constraint.anchor_b)
                joint_items.append(
                    dict(
                        kind=K_JOINT,
                        a=index_of[id(ca)],
                        b=index_of[id(cb)],
                        anchor_a=[float(delta_a[0]), float(delta_a[1])],
                        anchor_b=[float(delta_b[0]), float(delta_b[1])],
                        dist=float(constraint.dist),
                        rotate=bool(constraint.rotate),
                        fixed_rotation=None if per_env else float(fixed),
                        fixed_rotation_per_env=per_env,
                    )
                )
                if constraint.dist == 0:
                    continue
            if not _static_collides(world, ea, eb):
                continue
            ka, kb = _shape_kind(ea.shape), _shape_kind(eb.shape)
            if ka == SHAPE_SPHERE and kb == SHAPE_SPHERE:
                kind, first, second = K_SS, ia, ib
            elif {ka, kb} == {SHAPE_LINE, SHAPE_SPHERE}:
                kind = K_LS
                first, second = (ia, ib) if ka == SHAPE_LINE else (ib, ia)
            elif ka == SHAPE_LINE and kb == SHAPE_LINE:
                kind, first, second = K_LL, ia, ib
            elif {ka, kb} == {SHAPE_BOX, SHAPE_SPHERE}:
                kind = K_BS
                first, second = (ia, ib) if ka == SHAPE_BOX else (ib, ia)
            elif {ka, kb} == {SHAPE_BOX, SHAPE_LINE}:
                kind = K_BL
                first, second = (ia, ib) if ka == SHAPE_BOX else (ib, ia)
            elif ka == SHAPE_BOX and kb == SHAPE_BOX:
                kind, first, second = K_BB, ia, ib
            else:  # pragma: no cover - all 3x3 combos are handled above
                raise AssertionError()
            buckets[kind].append(dict(kind=kind, a=first, b=second))
    desc.items = joint_items + sum((buckets[k] for k in (K_SS, K_LS, K_LL, K_BS, K_BL, K_BB)), [])
    return desc


# ----------------------------------------------------------------------------------------
# tables
# ----------------------------------------------------------------------------------------
@dataclass
class PlanTables:
    desc: WorldDescription
    ent_f32: np.ndarray  # [E, EF_COLS]
    ent_i32: np.ndarray  # [E, EI_COLS]
    item_f32: np.ndarray  # [NI, IF_COLS]
    item_i32: np.ndarray  # [NI, II_COLS]
    inc_off: np.ndarray  # [E+1]   CSR offsets into inc
    inc: np.ndarray  # [..]    item*2 + side, ascending item order per entity
    n_joints: int
    n_masked: int  # items subject to the batch-wide broad-phase mask (line/box pairs)
    mask_slot: np.ndarray  # [NI] bit index in the pair mask, -1 if the item is always active
    spheres_only: bool = True  # every collision pair is sphere-sphere
    masked_items: np.ndarray = None  # [n_masked] item index of each mask bit

    def schedule(self, group: int):
        """Round-robin assignment of work items to the ``group`` lanes that own one env.

        Items of one kind are padded to a multiple of ``group`` so that every round is
        kind-uniform (no divergence inside a warp: all envs of a warp run the same table).
        Returns (sched [n_rounds, group] int32 item index or -1, round_kind [n_rounds]).
        """
        rows, kinds = [], []
        kinds_arr = self.item_i32[:, 0] if len(self.item_i32) else np.zeros((0,), np.int32)
        for kind in range(7):
            idx = np.nonzero(kinds_arr == kind)[0]
            for start in range(0, len(idx), group):
                chunk = idx[start : start + group]
                row = np.full((group,), -1, np.int32)
                row[: len(chunk)] = chunk
                rows.append(row)
                kinds.append(kind)
        if not rows:
            return np.zeros((0, group), np.int32), np.zeros((0,), np.int32)
        return np.stack(rows).astype(np.int32), np.asarray(kinds, np.int32)


def build_tables(desc: WorldDescription) -> PlanTables:
    E = desc.n_entities
    ent_f32 = np.zeros((max(E, 1), EF_COLS), np.float32)
    ent_i32 = np.zeros((max(E, 1), EI_COLS), np.int32)
    ent_flags: List[int] = []
    for i, e in enumerate(desc.entities):
        flags = 0
        flags |= F_MOVABLE if e["movable"] else 0
        flags |= F_ROTATABLE if e["rotatable"] else 0
        flags |= F_HOLLOW if e["hollow"] else 0
        flags |= F_AGENT if e["is_agent"] else 0
        row = ent_f32[i]
        row[EF_D0], row[EF_D1] = e["d0"], e["d1"]
        row[EF_MASS], row[EF_INERTIA] = e["mass"], e["inertia"]
        drag = e["drag"] if e["drag"] is not None else desc.drag
        row[EF_DRAG_MULT] = 1 - drag  # python double, rounded once (ref core.py:2866-2869)
        # friction: entity coefficient wins, else the world's if > 0 (ref core.py:2075-2102)
        lin = e["linear_friction"] if e["linear_friction"] is not None else (
            desc.linear_friction if desc.linear_friction > 0 else None
        )
        ang = e["angular_friction"] if e["angular_friction"] is not None else (
            desc.angular_friction if desc.angular_friction > 0 else None
        )
        if lin is not None:
            flags |= F_LIN_FRIC
            row[EF_LIN_FRIC] = lin
        if ang is not None:
            flags |= F_ANG_FRIC
            row[EF_ANG_FRIC] = ang
        if e["gravity"] is not None:
            flags |= F_GRAVITY
            row[EF_GRAV_X], row[EF_GRAV_Y] = e["gravity"]
        if e.get("gravity_per_env"):
            flags |= F_GRAVITY_ENV
        if e.get("mass_per_env"):
            flags |= F_MASS_ENV
            row[EF_INERTIA_K0], row[EF_INERTIA_K1] = inertia_constants(e["shape"], e["d0"], e["d1"])
        if e.get("lin_fric_per_env"):
            flags |= F_LIN_FRIC_ENV
        if e.get("ang_fric_per_env"):
            flags |= F_ANG_FRIC_ENV
        for name, col, bit in (
            ("max_speed", EF_MAX_SPEED, F_MAX_SPEED),
            ("v_range", EF_V_RANGE, F_V_RANGE),
            ("max_f", EF_MAX_F, F_MAX_F),
            ("f_range", EF_F_RANGE, F_F_RANGE),
            ("max_t", EF_MAX_T, F_MAX_T),
            ("t_range", EF_T_RANGE, F_T_RANGE),
        ):
            if e[name] is not None:
                flags |= bit
                row[col] = e[name]
        row[EF_CIRC_R] = e["circ_radius"]
        # is_overlapping(box, sphere) compares with fp32(radius + LINE_MIN_DIST), summed in double
        row[EF_R_PLUS_LMD] = e["d0"] + LINE_MIN_DIST
        if e["shape"] != SHAPE_SPHERE:
            flags |= F_TRIG
        ent_flags.append(flags)

    NI = len(desc.items)
    item_f32 = np.zeros((max(NI, 1), IF_COLS), np.float32)
    item_i32 = np.full((max(NI, 1), II_COLS), -1, np.int32)
    mask_slot = np.full((max(NI, 1),), -1, np.int32)
    lmd = np.float32(LINE_MIN_DIST)
    n_masked = 0
    spheres_only = True
    incident: List[List[int]] = [[] for _ in range(E)]
    for k, it in enumerate(desc.items):
        kind, a, b = it["kind"], it["a"], it["b"]
        ea, eb = desc.entities[a], desc.entities[b]
        flags = 0
        f = item_f32[k]
        if kind == K_JOINT:
            flags |= IFLAG_ALWAYS_ACTIVE
            flags |= IFLAG_JOINT_ROTATE if it["rotate"] else 0
            flags |= IFLAG_JOINT_ROT_PER_ENV if it["fixed_rotation_per_env"] else 0
            f[IF_AX], f[IF_AY] = it["anchor_a"]
            f[IF_BX], f[IF_BY] = it["anchor_b"]
            f[IF_DIST] = it["dist"]
            f[IF_FIXED_ROT] = 0.0 if it["fixed_rotation"] is None else it["fixed_rotation"]
        else:
            # batch-wide activation threshold: python-double sum, rounded once when compared
            # with the fp32 norm (ref core.py:2797-2799)
            f[IF_BROAD_THR] = ea["circ_radius"] + eb["circ_radius"]
            if kind == K_SS:
                # fp32(ra) + fp32(rb) (ref core.py:2327)
                f[IF_DMIN_BASE] = np.float32(ea["d0"]) + np.float32(eb["d0"])
                flags |= IFLAG_ALWAYS_ACTIVE  # mask is result-neutral for spheres
            else:
                spheres_only = False
                mask_slot[k] = n_masked
                n_masked += 1
                if kind == K_LS:  # a = line, b = sphere: fp32(r) + fp32(LMD) (ref core.py:2378)
                    f[IF_DMIN_BASE] = np.float32(eb["d0"]) + lmd
                elif kind == K_BS:  # a = box, b = sphere (ref core.py:2538)
                    f[IF_DMIN_BASE] = np.float32(eb["d0"]) + lmd
                else:  # L-L, B-L, B-B: LINE_MIN_DIST (+ inner-point depths at run time)
                    f[IF_DMIN_BASE] = lmd
        if kind == K_JOINT:
            ent_flags[a] |= F_TRIG
            ent_flags[b] |= F_TRIG
        item_i32[k] = (kind, a, b, flags | ((mask_slot[k] + 1) << 8))
        incident[a].append(2 * k)
        incident[b].append(2 * k + 1)

    for i, e in enumerate(desc.entities):
        ent_i32[i] = (e["shape"], ent_flags[i], e["agent_index"], 0)

    inc_off = np.zeros((E + 1,), np.int32)
    for i in range(E):
        inc_off[i + 1] = inc_off[i] + len(incident[i])
    inc = np.asarray(sum(incident, []), np.int32) if E else np.zeros((0,), np.int32)
    if inc.size == 0:
        inc = np.zeros((1,), np.int32)
    return PlanTables(
        desc=desc,
        ent_f32=ent_f32,
        ent_i32=ent_i32,
        item_f32=item_f32,
        item_i32=item_i32,
        inc_off=inc_off,
        inc=inc,
        n_joints=desc.n_joints,
        n_masked=n_masked,
        mask_slot=mask_slot,
        spheres_only=spheres_only,
        masked_items=(
            np.nonzero(mask_slot >= 0)[0].astype(np.int32) if n_masked else np.zeros((1,), np.int32)
        ),
    )


def algorithmic_bytes_per_env_substep(desc: WorldDescription) -> int:
    """Compulsory HBM traffic of one substep launch: 12*E + 24*M + 12*R + 12*A (SURVEY.md §8d)."""
    E = desc.n_entities
    M = sum(1 for e in desc.entities if e["movable"])
    R = sum(1 for e in desc.entities if e["rotatable"])
    A = desc.n_agents
    return 12 * E + 24 * M + 12 * R + 12 * A
