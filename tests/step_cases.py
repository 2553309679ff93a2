"""Worlds and per-env edge values for the per-entity phases of a substep (TEST INFRASTRUCTURE), shared by
tests/test_step_phases_hostsim.py (CPU) and tests/test_step_phases_gpu.py.

The worlds are built through this package's ``World`` / ``Agent`` / ``Landmark``; no entity collides, so they have
no work items and a substep is phase A then phase C.  One agent per clamp combination (``max_f``, ``f_range``, both;
``max_t``, ``t_range``, both; ``max_speed``, ``v_range``, both), entity and world friction and drag, world and entity
gravity, a movable agent that does not rotate, a rotatable agent that does not move, a movable landmark and a
rotatable one that does not move.  Variants: both semidims and 3 substeps, ``x_semidim`` only and 1 substep, every
range and semidim 0, and per-env masses, friction coefficients and gravity.

Each env row is one case: entity ``e`` of row ``b`` takes value ``(b + 7 e) mod n`` of each list, so every entity
meets every value.  The lists hold +-0, norms exactly at ``max_f`` / ``max_speed`` (3-4-5 multiples) and their fp32
neighbours, +-``f_range`` / ``v_range`` / ``t_range`` and their neighbours, +-inf, NaN, +-FLT_MAX, magnitudes whose
squares overflow or underflow, subnormals, one zero component, speeds at which ``|v| / sub_dt m`` equals the
friction cap ``coeff m``, and positions on, inside and outside each semidim.
"""
import math

import numpy as np
import torch

FLT_MAX = float(np.finfo(np.float32).max)
TINY = float(np.nextafter(np.float32(0), np.float32(1)))
SQ_OVER = 1.9e19  # x * x overflows fp32
SQ_UNDER = 1e-23  # x * x underflows to 0 in fp32
SUB = 1e-39  # a subnormal

MAX_F, F_RANGE, MAX_T, T_RANGE = 5.0, 0.8, 0.5, 0.4
MAX_SPEED, V_RANGE = 2.5, 1.5
LIN_FRIC, ANG_FRIC, WORLD_LIN, WORLD_ANG = 0.3, 0.25, 0.2, 0.15

VARIANTS = ("both_semidims_3", "x_semidim_1", "zero_ranges", "per_env")


def nxt(x, to):
    return float(np.nextafter(np.float32(x), np.float32(to)))


def _world_kwargs(variant):
    if variant == "both_semidims_3":
        return dict(substeps=3, drag=0.1, linear_friction=WORLD_LIN, angular_friction=WORLD_ANG,
                    gravity=(0.3, -0.7), x_semidim=1.0, y_semidim=0.5)
    if variant == "x_semidim_1":
        return dict(substeps=1, drag=0.25, x_semidim=0.8)
    if variant == "zero_ranges":
        return dict(substeps=2, drag=0.1, x_semidim=0.0, y_semidim=0.0)
    if variant == "per_env":
        return dict(substeps=2, drag=0.15, linear_friction=WORLD_LIN, gravity=(0.0, -0.4), x_semidim=2.0,
                    y_semidim=2.0)
    raise ValueError(variant)


def make_world(variant, B, device="cpu"):
    """(world, {entity index: {attribute: [B, 1] tensor}} per-env values, {entity index: [B, 2]} per-env gravity)."""
    from crafted import _ns

    ns = _ns("vectorizedmultiagentsimulator_b200")
    Agent, Landmark, World, Sphere = ns["Agent"], ns["Landmark"], ns["World"], ns["Sphere"]
    Rot = ns["HolonomicWithRotation"]
    world = World(B, device, dt=0.1, **_world_kwargs(variant))
    z = variant == "zero_ranges"
    fr, tr, vr = (0.0, 0.0, 0.0) if z else (F_RANGE, T_RANGE, V_RANGE)
    agents = [
        dict(max_f=MAX_F, max_t=MAX_T),
        dict(f_range=fr, t_range=tr),
        dict(max_f=MAX_F, f_range=fr, max_t=MAX_T, t_range=tr),
        dict(max_speed=MAX_SPEED),
        dict(v_range=vr),
        dict(max_speed=MAX_SPEED, v_range=vr),
        dict(linear_friction=LIN_FRIC, angular_friction=ANG_FRIC, drag=0.3, mass=2.0),
        dict(gravity=(0.1, -0.2), mass=0.5, rotatable=False, f_range=fr),
        dict(movable=False, t_range=tr, angular_friction=ANG_FRIC),
    ]
    for i, kw in enumerate(agents):
        kw.setdefault("rotatable", True)
        dyn = {"dynamics": Rot()} if kw["rotatable"] and kw.get("movable", True) else {}
        world.add_agent(Agent(name=f"agent_{i}", shape=Sphere(0.05), collide=False, **dyn, **kw))
    world.add_landmark(Landmark("crate", shape=Sphere(0.1), movable=True, rotatable=True, collide=False, mass=3.0,
                                angular_friction=0.05))
    world.add_landmark(Landmark("puck", shape=Sphere(0.04), movable=True, collide=False, linear_friction=0.1))
    world.add_landmark(Landmark("wheel", shape=Sphere(0.08), rotatable=True, collide=False))
    world.add_landmark(Landmark("post", shape=Sphere(0.03), collide=False))
    params, gravity = {}, {}
    if variant == "per_env":
        gen = torch.Generator().manual_seed(11)
        draw = lambda lo, hi, k=1: (torch.rand(B, k, generator=gen) * (hi - lo) + lo).to(device)  # noqa: E731
        byname = {e.name: i for i, e in enumerate(world.entities)}
        for name, attrs in (("agent_6", ("mass", "linear_friction", "angular_friction")), ("agent_3", ("mass",)),
                            ("crate", ("mass", "angular_friction")), ("puck", ("linear_friction",))):
            e = world.entities[byname[name]]
            for attr in attrs:
                v = draw(0.5, 3.0) if attr == "mass" else draw(0.02, 0.4)
                setattr(e, attr, v)
                params.setdefault(byname[name], {})[attr] = v
        for name in ("agent_4", "puck"):
            g = draw(-0.5, 0.5, 2)
            world.entities[byname[name]].gravity = g
            gravity[byname[name]] = g
    return world, params, gravity


def _pairs(r, at, comps=(3.0, 4.0)):
    """Vectors around a norm limit ``at`` (a 3-4-5 multiple) and a per-component range ``r``."""
    k = at / 5.0
    a, b = comps[0] * k, comps[1] * k
    out = [(0.0, 0.0), (-0.0, -0.0), (0.0, -0.0), (a, b), (a, nxt(b, math.inf)), (a, nxt(b, 0)), (-a, -b),
           (nxt(a, math.inf), -b), (b, -a)]
    if r:
        out += [(r, r), (-r, -r), (nxt(r, math.inf), nxt(-r, -math.inf)), (nxt(r, 0), -nxt(r, 0)), (r, 0.0),
                (-r, -0.0)]
    out += [(math.inf, 0.0), (-math.inf, 1.0), (math.nan, 0.5), (0.5, math.nan), (FLT_MAX, 0.0),
            (-FLT_MAX, FLT_MAX), (SQ_OVER, 0.0), (SQ_OVER, -SQ_OVER), (SQ_UNDER, 0.0), (SQ_UNDER, -SQ_UNDER),
            (SUB, -SUB), (TINY, 0.0), (0.0, -0.6), (0.4, 0.2), (2.0, -1.0), (-7.0, 0.3)]
    return out


def _scalars(limits):
    out = [0.0, -0.0, 0.1, -0.2, 1.0, math.inf, -math.inf, math.nan, FLT_MAX, -FLT_MAX, SQ_OVER, SQ_UNDER, SUB, TINY]
    for r in limits:
        if r:
            out += [r, -r, nxt(r, math.inf), nxt(-r, -math.inf), nxt(r, 0)]
    return out


def _cap_speeds(coeffs, sub_dt):
    """Speeds at which (|v| / sub_dt) m equals the friction cap coeff m, and their neighbours."""
    out = []
    for c in coeffs:
        v = float(np.float32(np.float32(c) * np.float32(sub_dt)))
        out += [v, nxt(v, math.inf), nxt(v, 0)]
    return out


def values(variant):
    """The edge-value lists of a variant: {"force": [(x, y)], "torque": [t], "vel": [(x, y)], "ang_vel": [w],
    "pos": [(x, y)], "rot": [r]}."""
    kw = _world_kwargs(variant)
    sub_dt = 0.1 / kw["substeps"]
    z = variant == "zero_ranges"
    caps = _cap_speeds([LIN_FRIC, 0.1, WORLD_LIN], sub_dt)
    ang_caps = _cap_speeds([ANG_FRIC, WORLD_ANG, 0.05], sub_dt)
    xs, ys = kw.get("x_semidim"), kw.get("y_semidim")
    pos = [(0.0, 0.0), (-0.0, 0.0), (0.3, -0.2), (math.inf, -math.inf), (math.nan, 0.0), (0.0, math.nan),
           (FLT_MAX, -FLT_MAX), (SUB, -0.0)]
    for s in (xs, ys):
        if s is not None:
            pos += [(s, s), (-s, -s), (nxt(s, math.inf), nxt(-s, -math.inf)), (nxt(s, 0), -nxt(s, 0)),
                    (2 * s + 0.5, -3 * s - 0.5)]
    return dict(
        force=_pairs(0.0 if z else F_RANGE, MAX_F),
        torque=_scalars([MAX_T] + ([] if z else [T_RANGE])),
        vel=_pairs(0.0 if z else V_RANGE, MAX_SPEED) + [(c, 0.0) for c in caps] + [(0.0, -c) for c in caps]
        + [(c, c) for c in caps[:3]],
        ang_vel=_scalars([]) + ang_caps + [-c for c in ang_caps],
        pos=pos,
        rot=[0.0, -0.0, 1.0, 3.0, -2.0, math.inf, math.nan, SUB, FLT_MAX],
    )


def batch(variant):
    """Number of env rows: the longest list, so every entity meets every value."""
    return max(len(v) for v in values(variant).values())


def state(variant, desc):
    """fp32 numpy state of the cases: pos / vel [B, E, 2], rot / ang_vel [B, E], force [B, A, 2], torque [B, A]."""
    vals = values(variant)
    B, E, A = batch(variant), desc.n_entities, desc.n_agents

    def fill(key, n, pair):
        lst = vals[key]
        out = np.zeros((B, n, 2) if pair else (B, n), np.float32)
        for b in range(B):
            for e in range(n):
                out[b, e] = lst[(b + 7 * e) % len(lst)]
        return out

    return dict(pos=fill("pos", E, True), vel=fill("vel", E, True), rot=fill("rot", E, False),
                ang_vel=fill("ang_vel", E, False), force=fill("force", A, True), torque=fill("torque", A, False))


def describe(variant):
    """(desc, tables, per-env values as numpy {attr: {entity: [B]}}, per-env gravity {entity: [B, 2]}, torch forms
    of both for the oracle)."""
    from vectorizedmultiagentsimulator_b200.simulator import plan as P

    world, params, gravity = make_world(variant, batch(variant))
    desc = P.describe_world(world)
    assert not desc.items
    env = {}
    for e, attrs in params.items():
        for attr, v in attrs.items():
            env.setdefault(attr, {})[e] = v.numpy().reshape(-1)
    return desc, P.build_tables(desc), env, {e: g.numpy() for e, g in gravity.items()}, params, gravity
