"""Float64 reference of the per-entity phases of a substep (TEST INFRASTRUCTURE), written in numpy from the formulas.

Phase A (ref core.py:1995-2102): the agent's action force clamped by ``max_f`` (norm) then ``f_range`` (per
component) and written back to its row, the torque likewise with ``max_t`` / ``t_range``, linear and angular
friction, world, entity and per-env gravity.  Phase C (ref core.py:2862-2908): semi-implicit Euler with drag on the
step's substep 0 only, ``max_speed`` (norm) then ``v_range``, then ``p + v sub_dt`` and the world's semidims.

Values carry a first-order bound on the error of an fp32 evaluation of the same chain of operations, in the
kernels' order (:class:`S`, action_ref's :class:`F` extended):

    F = ((0 + f_action) + friction) + m g_world + m g_entity + m g_env
    v = v drag_mult (substep 0) + (F / m) sub_dt;  max_speed;  v_range;  p = clamp(p + v sub_dt, semidim)

and the same for the rotation with the moment of inertia (per env: ``fp32(fp32(K0 m) K1)``, a parameter).

Where an fp32 branch decision may fall the other way within rounding (``n > max_f``, ``n > max_speed``,
``speed != 0``), the bound covers both branches (:func:`select`); ``min`` and the clamps are 1-Lipschitz and need
no such care.  Values an fp32 evaluation cannot approximate — a non-finite input or result, a magnitude past
FLT_MAX anywhere in the chain, the squares of a norm overflowing — are marked ``odd``: there the kernels are checked
against the fp32 oracle bit for bit instead.

``mistake`` keywords turn the reference into a plausible wrong implementation, to show the bound is tight enough to
catch it (tests/test_step_phases_hostsim.py).
"""
from __future__ import annotations

import numpy as np

from action_ref import F, U, f32

FLT_MAX = float(np.finfo(np.float32).max)
UNDER = 2.0 ** -150  # absolute rounding error of an fp32 result in the subnormal range
NORM_UNDER = 2.0 ** -74  # |sqrt(a) - sqrt(b)| for |a - b| <= 3 * 2^-150: the norm of vectors whose squares underflow

#: CUDA's approximate division and square root (the fast build: -prec-div=false, -prec-sqrt=false; CUDA C
#: Programming Guide, "Mathematical Functions": x / y 2 ulp, sqrtf 1 ulp) in place of correctly rounded ones
APPROX = False

MISTAKES = (
    "drag_every_substep", "drag_at_range_start", "max_speed_per_component", "v_range_before_max_speed",
    "semidim_before_update", "gravity_without_mass", "angular_friction_with_mass", "no_force_writeback",
)


class S(F):
    """:class:`F` whose roundings also admit the subnormal spacing, with a flag ``odd`` for values that have no
    meaningful float64 counterpart (propagated through every operation)."""

    __slots__ = ("odd",)

    def __init__(self, v, e=0.0, odd=False):
        super().__init__(v, e)
        with np.errstate(invalid="ignore", over="ignore"):
            bad = ~np.isfinite(self.v) | ~np.isfinite(self.e) | (np.abs(self.v) + self.e > FLT_MAX)
        self.odd = np.asarray(odd, dtype=bool) | bad

    @staticmethod
    def of(x):
        return x if isinstance(x, S) else S(f32(x))

    def _round(self, v, e):
        return S(v, e + U * np.abs(v) + UNDER)

    def __neg__(self):
        return S(-self.v, self.e, self.odd)

    def __abs__(self):
        return S(np.abs(self.v), self.e, self.odd)

    def __getitem__(self, k):
        return S(self.v[k], self.e[k], self.odd[k])

    def __rsub__(self, o):
        return S.of(o) - self

    def __rtruediv__(self, o):
        return S.of(o) / self


def _lift(name):
    def op(self, o):
        o = S.of(o)
        with np.errstate(all="ignore"):
            r = getattr(F, name)(self, o)
        r.odd = r.odd | self.odd | o.odd
        if APPROX and name == "__truediv__":
            r = S(r.v, r.e + 4 * U * np.abs(r.v), r.odd)
        return r

    return op


for _name in ("__add__", "__sub__", "__mul__", "__truediv__"):
    setattr(S, _name, _lift(_name))
S.__radd__, S.__rmul__ = S.__add__, S.__mul__


def zero(shape):
    return S(np.zeros(shape))


def select(cond, amb, a, b):
    """``where(cond, a, b)`` for an fp32 branch that may go the other way where ``amb``: there the bound covers the
    distance to either branch's value."""
    with np.errstate(invalid="ignore"):
        v = np.where(cond, a.v, b.v)
        e = np.where(cond, a.e, b.e)
        both = np.maximum(np.abs(v - a.v) + a.e, np.abs(v - b.v) + b.e)
    odd = np.where(cond, a.odd, b.odd) | (amb & (a.odd | b.odd))
    return S(v, np.where(amb, np.maximum(e, both), e), odd)


def clip(x, lo, hi):
    """torch.clamp: NaN stays NaN; 1-Lipschitz, so the bound carries through."""
    return S(np.clip(x.v, lo, hi), x.e, x.odd)


def norm2(x, y):
    """fp32 ``sqrt(fma(y, y, x * x))``: the norm is 1-Lipschitz in its inputs, its three roundings add 2U;
    squares in the subnormal range add NORM_UNDER; squares past FLT_MAX make the value odd (fp32 gives inf)."""
    with np.errstate(all="ignore"):
        sq = x.v * x.v + y.v * y.v
        v = np.sqrt(sq)
        e = np.hypot(x.e, y.e) + (4.0 if APPROX else 2.0) * U * v + np.where(sq < 2.0 ** -125, NORM_UNDER, 0.0)
    return S(v, e, x.odd | y.odd | (sq > FLT_MAX * (1 - 4 * U)))


def norm(comps):
    """torch.linalg.vector_norm over the last dim: ``norm2`` of a pair; ``|x|`` of one element, exact (no square
    to overflow or underflow)."""
    return norm2(*comps) if len(comps) > 1 else abs(comps[0])


def clamp_norm(comps, mx, per_component=False):
    """clamp_with_norm (ref utils.py:168-173): rescale to ``mx`` where the norm exceeds it."""
    mx = float(f32(mx))
    if per_component:
        return [clip(c, -mx, mx) for c in comps]
    n = norm(comps)
    cond = n.v > mx
    amb = (np.abs(n.v - mx) <= n.e) & (n.e > 0)
    return [select(cond, amb, (c / n) * mx, c) for c in comps]


def friction(comps, coeff, m, sub_dt):
    """ref core.py:2055-2073 per component: ``-(v / |v|) min(coeff m, (|v| / sub_dt) m)`` where |v| != 0."""
    shape = comps[0].v.shape
    speed = norm(comps)
    cap = S.of(coeff) * m
    loose = speed.e >= speed.v / 2  # direction unknown: both fp32 and float64 components lie in [-1, 1]
    out = []
    for c in comps:
        d = -(c / speed)
        d = S(d.v, np.where(loose, np.minimum(d.e, 2.0 + 4 * U), d.e), d.odd)
        lim = (abs(c) / sub_dt) * m
        with np.errstate(invalid="ignore"):
            mn = S(np.minimum(cap.v, lim.v), np.maximum(cap.e, lim.e), cap.odd | lim.odd)
        out.append(d * mn)
    cond = speed.v != 0
    amb = speed.v <= speed.e
    return [select(cond, amb, f, zero(shape)) for f in out]


def entity_constants(desc, tables, env=None):
    """Per entity: (mass, inertia, linear, angular friction coefficient or None) as float64 arrays/scalars of their
    fp32 values.  ``env``: {"mass" | "linear_friction" | "angular_friction": {entity: [B]}} per-env values."""
    from vectorizedmultiagentsimulator_b200.simulator import plan as P

    env = env or {}
    out = []
    for i, e in enumerate(desc.entities):
        if e.get("mass_per_env"):
            m32 = np.asarray(env["mass"][i], np.float32)
            k0, k1 = tables.ent_f32[i, P.EF_INERTIA_K0], tables.ent_f32[i, P.EF_INERTIA_K1]
            mass, inertia = f32(m32), f32((k0 * m32) * k1)
        else:
            mass, inertia = f32(e["mass"]), f32(e["inertia"])
        lin = env["linear_friction"][i] if e.get("lin_fric_per_env") else e["linear_friction"]
        ang = env["angular_friction"][i] if e.get("ang_fric_per_env") else e["angular_friction"]
        if lin is None and desc.linear_friction > 0:
            lin = desc.linear_friction
        if ang is None and desc.angular_friction > 0:
            ang = desc.angular_friction
        out.append((mass, inertia, None if lin is None else f32(lin), None if ang is None else f32(ang)))
    return out


def substeps(desc, tables, state, first=0, n=None, env=None, gravity=None, **mistake):
    """Substeps ``first .. first + n - 1`` of a world without work items.  ``state``: fp32 arrays ``pos`` / ``vel``
    [B, E, 2], ``rot`` / ``ang_vel`` [B, E], ``force`` [B, A, 2], ``torque`` [B, A]; ``env`` as in
    :func:`entity_constants`, ``gravity``: {entity: [B, 2]} per-env gravity.  Returns the same keys as :class:`S`."""
    assert not desc.items, "the reference covers the per-entity phases only"
    assert all(k in MISTAKES for k in mistake), mistake
    n = desc.substeps if n is None else n
    sub_dt = float(f32(desc.dt / desc.substeps))
    E = desc.n_entities
    st = {k: S(f32(v)) for k, v in state.items()}
    pos = [[st["pos"][:, e, 0], st["pos"][:, e, 1]] for e in range(E)]
    vel = [[st["vel"][:, e, 0], st["vel"][:, e, 1]] for e in range(E)]
    rot = [st["rot"][:, e] for e in range(E)]
    ang = [st["ang_vel"][:, e] for e in range(E)]
    force = [[st["force"][:, j, 0], st["force"][:, j, 1]] for j in range(st["force"].v.shape[1])]
    torque = [st["torque"][:, j] for j in range(st["torque"].v.shape[1])]
    consts = entity_constants(desc, tables, env)
    g_world = [float(f32(g)) for g in desc.gravity]
    has_world_gravity = any(g != 0.0 for g in desc.gravity)
    shape = st["rot"].v.shape[:1]

    def gravity_term(m, g):
        return S.of(g) if mistake.get("gravity_without_mass") else m * g

    for s in range(first, first + n):
        Fs, Ts = [], []
        for i, e in enumerate(desc.entities):  # phase A
            m, inertia, lin, angc = S.of(consts[i][0]), S.of(consts[i][1]), consts[i][2], consts[i][3]
            Fx, Fy, T = zero(shape), zero(shape), zero(shape)
            if e["is_agent"]:
                j = e["agent_index"]
                if e["movable"]:
                    f = force[j]
                    if e["max_f"] is not None:
                        f = clamp_norm(f, e["max_f"])
                    if e["f_range"] is not None:
                        r = float(f32(e["f_range"]))
                        f = [clip(c, -r, r) for c in f]
                    if not mistake.get("no_force_writeback"):
                        force[j] = f
                    Fx, Fy = Fx + f[0], Fy + f[1]
                if e["rotatable"]:
                    t = [torque[j]]
                    if e["max_t"] is not None:
                        t = clamp_norm(t, e["max_t"])
                    if e["t_range"] is not None:
                        r = float(f32(e["t_range"]))
                        t = [clip(t[0], -r, r)]
                    if not mistake.get("no_force_writeback"):
                        torque[j] = t[0]
                    T = T + t[0]
            if lin is not None:
                fx, fy = friction(vel[i], lin, m, sub_dt)
                Fx, Fy = Fx + fx, Fy + fy
            if angc is not None:
                (tf,) = friction([ang[i]], angc, m if mistake.get("angular_friction_with_mass") else inertia, sub_dt)
                T = T + tf
            if e["movable"]:
                if has_world_gravity:
                    Fx, Fy = Fx + gravity_term(m, g_world[0]), Fy + gravity_term(m, g_world[1])
                if e["gravity"] is not None:
                    gx, gy = (float(f32(g)) for g in e["gravity"])
                    Fx, Fy = Fx + gravity_term(m, gx), Fy + gravity_term(m, gy)
                if e.get("gravity_per_env"):
                    g = f32(np.asarray(gravity[i], np.float32))
                    Fx, Fy = Fx + gravity_term(m, g[:, 0]), Fy + gravity_term(m, g[:, 1])
            Fs.append((Fx, Fy))
            Ts.append(T)
        drag_now = s == 0
        if mistake.get("drag_every_substep"):
            drag_now = True
        if mistake.get("drag_at_range_start"):
            drag_now = s == first
        for i, e in enumerate(desc.entities):  # phase C
            m, inertia = (S.of(c) for c in consts[i][:2])
            drag = e["drag"] if e["drag"] is not None else desc.drag
            drag_mult = float(f32(1 - drag))
            if e["movable"]:
                v = vel[i]
                if drag_now:
                    v = [c * drag_mult for c in v]
                v = [c + (Fc / m) * sub_dt for c, Fc in zip(v, Fs[i])]
                speed_first = not mistake.get("v_range_before_max_speed")
                for stage in ("max_speed", "v_range") if speed_first else ("v_range", "max_speed"):
                    if stage == "max_speed" and e["max_speed"] is not None:
                        v = clamp_norm(v, e["max_speed"], per_component=mistake.get("max_speed_per_component"))
                    if stage == "v_range" and e["v_range"] is not None:
                        r = float(f32(e["v_range"]))
                        v = [clip(c, -r, r) for c in v]
                semis = [desc.x_semidim, desc.y_semidim]
                p = pos[i]
                if mistake.get("semidim_before_update"):
                    p = [c if sd is None else clip(c, -float(f32(sd)), float(f32(sd))) for c, sd in zip(p, semis)]
                    p = [c + vc * sub_dt for c, vc in zip(p, v)]
                else:
                    p = [c + vc * sub_dt for c, vc in zip(p, v)]
                    p = [c if sd is None else clip(c, -float(f32(sd)), float(f32(sd))) for c, sd in zip(p, semis)]
                vel[i], pos[i] = v, p
            if e["rotatable"]:
                w = ang[i]
                if drag_now:
                    w = w * drag_mult
                w = w + (Ts[i] / inertia) * sub_dt
                ang[i] = w
                rot[i] = rot[i] + w * sub_dt

    def pack(rows, pairs):
        if pairs:
            v = np.stack([np.stack([r[0].v, r[1].v], -1) for r in rows], 1)
            e = np.stack([np.stack([r[0].e, r[1].e], -1) for r in rows], 1)
            o = np.stack([np.stack([r[0].odd, r[1].odd], -1) for r in rows], 1)
        else:
            v, e, o = (np.stack([getattr(r, k) for r in rows], 1) for k in ("v", "e", "odd"))
        return S(v, e, o)

    return dict(pos=pack(pos, True), vel=pack(vel, True), rot=pack(rot, False), ang_vel=pack(ang, False),
                force=pack(force, True), torque=pack(torque, False))
