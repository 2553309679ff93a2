"""One ``World.step`` on CPU for worlds whose entities carry per-env physical parameters (TEST INFRASTRUCTURE).

``oracle.world_step.world_step`` with the per-entity phase and the integration of the reference restated
for ``[B, 1]`` masses and friction coefficients (ref core.py:2043-2102, 2862-2908): a per-env mass
broadcasts through gravity, the friction cap and the integration, and the moment of inertia is
``shape.moment_of_inertia(mass)`` on the tensor (ref core.py:123-124, 160-161, 187-188), i.e.
``fl(fl(K0 * m) * K1)`` with the plan's fp32 constants.  The joints and contacts are the oracle's own
functions.  ``tests/test_entity_params.py`` pins this against the reference's recorded roll-out.
"""
from typing import Dict, Optional

import torch

from oracle import world_step as WS
from vectorizedmultiagentsimulator_b200.simulator import plan as P


def _friction(vel, coeff, mass, sub_dt):
    """ref core.py:2055-2073 with ``coeff`` a python number or a ``[B, 1]`` tensor, ``mass`` likewise."""
    speed = torch.linalg.vector_norm(vel, dim=-1)
    static = speed == 0
    coeff_t = coeff.expand(vel.shape) if isinstance(coeff, torch.Tensor) else torch.full_like(vel, coeff)
    cap = coeff_t * mass
    f = -(vel / torch.where(static, 1e-8, speed).unsqueeze(-1)) * torch.minimum(cap, (vel.abs() / sub_dt) * mass)
    return torch.where(static.unsqueeze(-1).expand(vel.shape), 0.0, f)


def entity_params(tables: P.PlanTables, params: Dict[int, Dict[str, torch.Tensor]]):
    """Per entity: (mass, moment of inertia, linear-friction coefficient, angular-friction coefficient), each a
    python float or a ``[B, 1]`` tensor; ``params``: {entity index: {"mass" | "linear_friction" |
    "angular_friction": [B, 1]}}."""
    desc = tables.desc
    out = []
    for i, e in enumerate(desc.entities):
        p = params.get(i, {})
        mass, inertia = e["mass"], e["inertia"]
        if e.get("mass_per_env"):
            mass = p["mass"]
            k0 = torch.tensor(tables.ent_f32[i, P.EF_INERTIA_K0], dtype=torch.float32)
            k1 = torch.tensor(tables.ent_f32[i, P.EF_INERTIA_K1], dtype=torch.float32)
            inertia = (k0 * mass) * k1
        lin = p["linear_friction"] if e.get("lin_fric_per_env") else e["linear_friction"]
        ang = p["angular_friction"] if e.get("ang_fric_per_env") else e["angular_friction"]
        out.append((mass, inertia, lin, ang))
    return out


def world_step(
    tables: P.PlanTables,
    state: Dict[str, torch.Tensor],
    params: Dict[int, Dict[str, torch.Tensor]],
    fixed_rot: Optional[Dict[int, torch.Tensor]] = None,
    ent_gravity: Optional[Dict[int, torch.Tensor]] = None,
    exact_broad_phase: bool = True,
) -> None:
    """Advance ``state`` in place by one step (all substeps)."""
    desc = tables.desc
    pos, vel, rot, ang_vel = state["pos"], state["vel"], state["rot"], state["ang_vel"]
    force_in, torque_in = state["force"], state["torque"]
    B, E = pos.shape[0], desc.n_entities
    sub_dt = desc.dt / desc.substeps
    g_world = torch.tensor(desc.gravity, dtype=torch.float32)
    has_world_gravity = bool((g_world != 0).any())
    ent = entity_params(tables, params)

    for s in range(desc.substeps):
        F = [torch.zeros(B, 2, dtype=torch.float32) for _ in range(E)]
        T = [torch.zeros(B, 1, dtype=torch.float32) for _ in range(E)]
        for i, e in enumerate(desc.entities):
            mass, inertia, lin, ang = ent[i]
            if e["is_agent"]:
                j = e["agent_index"]
                if e["movable"]:
                    f = force_in[:, j]
                    if e["max_f"] is not None:
                        f = WS.clamp_with_norm(f, e["max_f"])
                    if e["f_range"] is not None:
                        f = torch.clamp(f, -e["f_range"], e["f_range"])
                    force_in[:, j] = f
                    F[i] = F[i] + f
                if e["rotatable"]:
                    t = torque_in[:, j : j + 1]
                    if e["max_t"] is not None:
                        t = WS.clamp_with_norm(t, e["max_t"])
                    if e["t_range"] is not None:
                        t = torch.clamp(t, -e["t_range"], e["t_range"])
                    torque_in[:, j : j + 1] = t
                    T[i] = T[i] + t
            if lin is None and desc.linear_friction > 0:
                lin = desc.linear_friction
            if lin is not None:
                F[i] = F[i] + _friction(vel[:, i], lin, mass, sub_dt)
            if ang is None and desc.angular_friction > 0:
                ang = desc.angular_friction
            if ang is not None:
                T[i] = T[i] + _friction(ang_vel[:, i : i + 1], ang, inertia, sub_dt)
            if e["movable"]:
                if has_world_gravity:
                    F[i] = F[i] + mass * g_world
                if e["gravity"] is not None:
                    F[i] = F[i] + mass * torch.tensor(e["gravity"], dtype=torch.float32)
                if e.get("gravity_per_env"):
                    F[i] = F[i] + mass * ent_gravity[i]

        for kind in (P.K_JOINT, P.K_SS, P.K_LS, P.K_LL, P.K_BS, P.K_BL, P.K_BB):
            items = [k for k, it in enumerate(desc.items) if it["kind"] == kind]
            if kind != P.K_JOINT and exact_broad_phase and items:
                items = [k for k, on in zip(items, WS.broad_phase_active_many(tables, items, pos)) if on]
            if not items:
                continue
            if kind == P.K_JOINT:
                results = WS._joint_bucket(tables, items, pos, rot, fixed_rot)
            else:
                results = WS._contact_bucket(tables, kind, items, pos, rot)
            for k in items:
                a, b = desc.items[k]["a"], desc.items[k]["b"]
                fa, ta, fb, tb = results[k]
                ea, eb = desc.entities[a], desc.entities[b]
                if ea["movable"]:
                    F[a] = F[a] + fa
                if ea["rotatable"] and ta is not None:
                    T[a] = T[a] + ta
                if eb["movable"]:
                    F[b] = F[b] + fb
                if eb["rotatable"] and tb is not None:
                    T[b] = T[b] + tb

        for i, e in enumerate(desc.entities):
            mass, inertia, _, _ = ent[i]
            drag = e["drag"] if e["drag"] is not None else desc.drag
            if e["movable"]:
                v = vel[:, i]
                if s == 0:
                    v = v * (1 - drag)
                v = v + (F[i] / mass) * sub_dt
                if e["max_speed"] is not None:
                    v = WS.clamp_with_norm(v, e["max_speed"])
                if e["v_range"] is not None:
                    v = v.clamp(-e["v_range"], e["v_range"])
                p = pos[:, i] + v * sub_dt
                px, py = p[..., 0], p[..., 1]
                if desc.x_semidim is not None:
                    px = px.clamp(-desc.x_semidim, desc.x_semidim)
                if desc.y_semidim is not None:
                    py = py.clamp(-desc.y_semidim, desc.y_semidim)
                vel[:, i] = v
                pos[:, i] = torch.stack([px, py], dim=-1)
            if e["rotatable"]:
                w = ang_vel[:, i : i + 1]
                if s == 0:
                    w = w * (1 - drag)
                w = w + (T[i] / inertia) * sub_dt
                ang_vel[:, i : i + 1] = w
                rot[:, i : i + 1] = rot[:, i : i + 1] + w * sub_dt
