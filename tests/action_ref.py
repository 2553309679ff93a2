"""Float64 reference of the action ingest (TEST INFRASTRUCTURE): the decoding of continuous, discrete and
multi-discrete actions and the kinematic action models, written in numpy from the formulas.

Every function returns a value and, where the fp32 result is not exact, a first-order bound on the error of an
fp32 evaluation of the same chain of operations (:class:`F`):

* each fp32 ``+ - * /`` adds ``2^-24 |result|`` and carries its inputs' bounds through the partial derivatives;
* ``sin`` / ``cos`` / ``tan`` / ``atan2`` add their documented maximum error in ulp, the larger of CUDA's (CUDA C
  Programming Guide, "Mathematical Functions": 2, 2, 4 and 3 ulp) and glibc's (1 or 2 ulp), so the same bound
  serves the GPU and the g++ build of the device code;
* parameters enter as their fp32 values with error 0 (``F.param``).

Reference formulas (vmas/simulator/...): environment/environment.py:616-655 (NaN assertion before the clamp,
the clamp, the range assertion after it, ``u = action * u_multiplier``) and :656-707 (the flat index unravelled
with ``//`` and ``%``, the odd-n re-ordering, ``(k / (n - 1)) * 2 u_max - u_max``); dynamics/holonomic.py:14-15,
holonomic_with_rot.py, forward.py, roatation.py; dynamics/diff_drive.py:27-82, kinematic_bicycle.py:38-111 and
drone.py:59-166 (the ODE, Euler or classic RK4, and the back-solve ``m (delta - v dt) / dt^2``).
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24  # unit roundoff of fp32
ULP = dict(sin=2, cos=2, tan=4, atan2=3)


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def _ulp(v):
    return np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


class F:
    """A float64 value ``v`` with a bound ``e`` on |fp32 evaluation - v| (numpy arrays, broadcast)."""

    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.broadcast_to(np.asarray(e, dtype=np.float64), self.v.shape)

    @staticmethod
    def param(x):
        """A parameter or an fp32 input: its fp32 value, exact."""
        return F(f32(x))

    @staticmethod
    def of(x):
        return x if isinstance(x, F) else F.param(x)

    def _round(self, v, e):
        return F(v, e + U * np.abs(v))

    def __add__(self, o):
        o = F.of(o)
        return self._round(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = F.of(o)
        return self._round(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return F.of(o) - self

    def __mul__(self, o):
        o = F.of(o)
        return self._round(self.v * o.v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = F.of(o)
        v = self.v / o.v
        return self._round(v, (self.e + np.abs(v) * o.e) / np.maximum(np.abs(o.v) - o.e, np.abs(o.v) / 2))

    def __rtruediv__(self, o):
        return F.of(o) / self

    def __neg__(self):
        return F(-self.v, self.e)

    def __getitem__(self, k):
        return F(self.v[k], self.e[k])


def _fn(name, v, slope, x):
    return F(v, slope * x.e + ULP[name] * _ulp(v))


def sin(x):
    return _fn("sin", np.sin(x.v), np.abs(np.cos(x.v)), x)


def cos(x):
    return _fn("cos", np.cos(x.v), np.abs(np.sin(x.v)), x)


def tan(x):
    t = np.tan(x.v)
    return _fn("tan", t, 1.0 + t * t, x)


def atan2_1(y):
    """atan2(y, 1)"""
    return _fn("atan2", np.arctan2(y.v, 1.0), 1.0 / (1.0 + y.v * y.v), y)


def clamp(x, lo, hi):
    return F(np.clip(x.v, lo, hi), x.e)


def stack(parts):
    return F(np.stack([p.v for p in parts], -1), np.stack([p.e for p in parts], -1))


# ---- continuous actions --------------------------------------------------------------------------------------------
def continuous(actions, u_range, u_mult, clamp_actions: bool):
    """``actions`` fp32 [B, n], ``u_range`` / ``u_mult`` [n].  Returns (u fp32 [B, n], flagged bool [B]).  u is exact:
    the product of two fp32 numbers is exact in float64, so one rounding to fp32 is the fp32 product."""
    a = np.asarray(actions, dtype=np.float32).astype(np.float64)
    r, m = f32(u_range), f32(u_mult)
    c = np.clip(a, -r, r) if clamp_actions else a  # np.clip, like torch.clamp, keeps NaN
    with np.errstate(invalid="ignore"):
        flagged = np.isnan(a).any(-1) | (np.abs(c) > r).any(-1)
        u = (c * m).astype(np.float32)
    return u, flagged


def holonomic(u):
    """(force [B, 2], torque [B] or None) of Holonomic (2 components) / HolonomicWithRotation (3); exact."""
    return u[:, :2], (u[:, 2] if u.shape[1] > 2 else None)


def forward(u0, rot):
    th = F.param(rot)
    u = F.param(u0)
    return u * cos(th), u * sin(th)


# ---- discrete actions ----------------------------------------------------------------------------------------------
def unravel(flat, nvec):
    """Per-component indices of the flat index (the reference's floor ``//`` and ``%``), [B, len(nvec)] int64."""
    flat = np.asarray(flat, dtype=np.int64).reshape(-1)
    parts = []
    for i in range(len(nvec)):
        stride = math.prod(nvec[i + 1:])
        parts.append(flat // stride)
        flat = flat % stride
    return np.stack(parts, -1)


def discrete(idx, nvec, u_range, u_mult):
    """``idx`` int64 [B, n] per-component indices.  Returns (u as F [B, n], the fp32 op chain evaluated with numpy
    float32 [B, n], flagged [B])."""
    idx = np.asarray(idx, dtype=np.int64)
    n = np.asarray(nvec, dtype=np.int64)
    flagged = ((idx < 0) | (idx >= n)).any(-1)
    k = idx.copy()
    odd = (n % 2) != 0
    stay = odd & (k == 0)
    lower = odd & (k > 0) & (k <= n // 2)
    k = np.where(stay, n // 2, np.where(lower, k - 1, k))
    r, m = f32(u_range), f32(u_mult)
    kf = F(f32(k), np.abs(f32(k) - k))  # the int -> fp32 conversion rounds above 2^24
    u = ((kf / f32(n - 1)) * (2 * r) - r) * m
    # the same chain in fp32
    k32, n32 = k.astype(np.float32), (n - 1).astype(np.float32)
    r32, m32 = r.astype(np.float32), m.astype(np.float32)
    chain = ((k32 / n32) * (np.float32(2) * r32) - r32) * m32
    return u, chain, flagged


# ---- kinematic models ----------------------------------------------------------------------------------------------
def _integrate(f, s0, dt, rk4):
    """delta of the ODE s' = f(s) over dt: Euler or classic RK4, the reference's order of operations."""
    k1 = f(s0)
    if not rk4:
        return [dt * k for k in k1]
    k2 = f([s + dt * k / 2 for s, k in zip(s0, k1)])
    k3 = f([s + dt * k / 2 for s, k in zip(s0, k2)])
    k4 = f([s + dt * k for s, k in zip(s0, k3)])
    w = dt / 6
    return [w * (a + 2 * b + 2 * c + d) for a, b, c, d in zip(k1, k2, k3, k4)]


def back_solve(d, vel, ang_vel, dt, mass, inertia, dt2_wrong=False):
    """Force and torque that realise the pose change ``d`` = (dx, dy, dyaw) under the world's semi-implicit Euler
    step.  dt^2: the kernels round fp32(dt) * fp32(dt), torch rounds the double dt**2 once; the two differ by
    up to 3 * 2^-24 dt^2, which the bound admits."""
    dt = F.param(dt)
    dt2 = dt if dt2_wrong else F(dt.v * dt.v, 3 * U * dt.v * dt.v)
    vx, vy, w = F.param(vel[:, 0]), F.param(vel[:, 1]), F.param(ang_vel)
    fx = mass * ((d[0] - vx * dt) / dt2)
    fy = mass * ((d[1] - vy * dt) / dt2)
    tq = inertia * ((d[2] - w * dt) / dt2)
    return fx, fy, tq


def diff_drive(u, rot, vel, ang_vel, dt, mass, inertia, rk4, **mistake):
    """u fp32 [B, 2] (decoded), rot [B], vel [B, 2], ang_vel [B].  Returns (fx, fy, torque) as F."""
    v, w = F.param(u[:, 0]), F.param(u[:, 1])
    rk4 = rk4 and not mistake.get("euler")

    def f(s):
        return [v * cos(s[2]), v * sin(s[2]), w]

    zero = F(np.zeros_like(np.asarray(rot, np.float64)))
    d = _integrate(f, [zero, zero, F.param(rot)], F.param(dt), rk4)
    return back_solve(d, vel, ang_vel, dt, F.param(mass), F.param(inertia), mistake.get("dt2"))


def bicycle(u, rot, vel, ang_vel, dt, mass, inertia, rk4, l_f, l_r, max_steer, **mistake):
    v = F.param(u[:, 0])
    steer = F.param(u[:, 1])
    if not mistake.get("no_steer_clamp"):
        lim = f32(max_steer)
        steer = clamp(steer, -lim, lim)
    lf, lr = F.param(l_f), F.param(l_r)
    wheelbase = lf + lr
    t = tan(steer)
    slip = F(np.zeros_like(t.v)) if mistake.get("no_slip") else atan2_1(t * lr / wheelbase)
    rk4 = rk4 and not mistake.get("euler")

    def f(s):
        h = s[2] + slip
        return [v * cos(h), v * sin(h), v / wheelbase * cos(slip) * t]

    zero = F(np.zeros_like(np.asarray(rot, np.float64)))
    d = _integrate(f, [zero, zero, F.param(rot)], F.param(dt), rk4)
    return back_solve(d, vel, ang_vel, dt, F.param(mass), F.param(inertia), mistake.get("dt2"))


def drone(u, rot, pos, vel, ang_vel, state, dt, mass, inertia, rk4, I, g=9.81, **mistake):
    """u fp32 [B, 4], state fp32 [B, 12].  Returns (u with the thrust offset, new 12-state, fx, fy, torque) as F.
    The force comes from delta[6], delta[7] (velocity changes) and the torque from delta[5] (yaw-rate change): the
    reference's own choice of components (drone.py:150-154)."""
    m = F.param(mass)
    thrust = F.param(u[:, 0])
    if not mistake.get("no_thrust_offset"):
        thrust = thrust + m * F.param(g)
    tx, ty, tz = (F.param(u[:, j]) for j in (1, 2, 3))
    Ixx, Iyy, Izz = (F.param(x) for x in I)
    s0 = [F.param(state[:, j]) for j in range(12)]
    s0[9], s0[10] = F.param(pos[:, 0]), F.param(pos[:, 1])
    if not mistake.get("yaw_not_from_rot"):
        s0[2] = F.param(rot)
    grav = F.param(g)

    def f(s):
        sr, cr, sp, cp, sy, cy = sin(s[0]), cos(s[0]), sin(s[1]), cos(s[1]), sin(s[2]), cos(s[2])
        p, q, r = s[3], s[4], s[5]
        return [
            p, q, r,
            (tx - (Iyy - Izz) * q * r) / Ixx,
            (ty - (Izz - Ixx) * p * r) / Iyy,
            (tz - (Ixx - Iyy) * p * q) / Izz,
            (cr * sp * cy + sr * sy) * thrust / m,
            (cr * sp * sy - sr * cy) * thrust / m,
            (cr * cp) * thrust / m - grav,
            s[6], s[7], s[8],
        ]

    d = _integrate(f, s0, F.param(dt), rk4 and not mistake.get("euler"))
    new_state = stack([a + b for a, b in zip(s0, d)])
    fx, fy, tq = back_solve((d[6], d[7], d[5]), vel, ang_vel, dt, m, F.param(inertia), mistake.get("dt2"))
    u_out = stack([thrust, tx, ty, tz])
    return u_out, new_state, fx, fy, tq
