"""The action-ingest cases shared by tests/test_action_ingest_hostsim.py (CPU) and tests/test_action_ingest_gpu.py
(TEST INFRASTRUCTURE): edge values of continuous actions, discrete index sets, kinematic-model states and
commands, and a small scenario whose agents carry chosen ranges, multipliers and action models."""
import math

import numpy as np
import torch

RANGES = [1.0, 0.7, 1e-4, 3.0]
MULTS = [1.0, 0.7, 0.01]
FLT_MAX = float(np.finfo(np.float32).max)
TINY = float(np.nextafter(np.float32(0), np.float32(1)))  # the smallest subnormal


def _next(x, to):
    return float(np.nextafter(np.float32(x), np.float32(to)))


def edge_values(r):
    """(legal with clamping off, legal only with clamping on, never legal) fp32 values of a component of range r."""
    r = float(np.float32(r))
    legal = [0.0, -0.0, r, -r, _next(r, 0), _next(-r, 0), TINY, -TINY]
    clamped = [_next(r, math.inf), _next(-r, -math.inf), math.inf, -math.inf, FLT_MAX, -FLT_MAX]
    return legal, clamped, [math.nan]


def agent_layouts():
    """[(u_range, u_multiplier)] of the continuous agents: every range with every multiplier, and one agent with the
    maximum action size of 8."""
    out = []
    for k in range(len(MULTS)):
        out.append((RANGES, [MULTS[(k + j) % len(MULTS)] for j in range(len(RANGES))]))
    out.append((RANGES + RANGES[::-1], [MULTS[j % len(MULTS)] for j in range(8)]))
    return out


def legal_batch(u_range, clamp, B, rng):
    """[B, n] fp32: every legal edge value of each component, then random values in range."""
    n = len(u_range)
    a = (rng.random((B, n)) * 2 - 1) * np.asarray(u_range)
    for j, r in enumerate(u_range):
        legal, clamped, _ = edge_values(r)
        vals = legal + (clamped if clamp else [])
        for i, v in enumerate(vals):
            a[(i + 3 * j) % B, j] = v
    return a.astype(np.float32)


def bad_values(r, clamp):
    legal, clamped, nan = edge_values(r)
    return nan if clamp else clamped + nan


DISCRETE_N = [2, 3, 4, 5, 1000, 1001]
BIG_N = 2 ** 24 + 1
MULTI_NVEC = [[3, 4], [5, 2, 3]]


def discrete_indices(n):
    """Every index of a small n, the end points (and the middle) of a large one."""
    if n <= 8:
        return list(range(n))
    return [0, 1, 2, n // 2 - 1, n // 2, n // 2 + 1, n - 2, n - 1]


YAWS = [0.0, math.pi, -math.pi, math.pi / 2, -math.pi / 2, 1e3, -1e4]
DTS = [0.1, 0.005]


def kinematic_cases(kind, rng, u_range):
    """(u [B, size] decoded commands, rot [B], ang_vel [B], drone state [B, 12] or None) for one model: every yaw with
    zero, +-range and random commands."""
    rows, states = [], []
    for yaw in YAWS:
        if kind == "diff":
            cmds = [(0.0, 0.0), (u_range[0], 0.0), (-u_range[0], u_range[1]), (u_range[0], -u_range[1])]
            cmds += [tuple((rng.random(2) * 2 - 1) * u_range) for _ in range(2)]
        elif kind == "bicycle":
            # steering 0, +-max and beyond +-max (clamped); u_range[1] is beyond the steering limit
            cmds = [(u_range[0], 0.0), (-u_range[0], 1.4), (u_range[0], -1.4), (0.5 * u_range[0], u_range[1]),
                    (u_range[0], -u_range[1]), (0.0, 0.3)]
        else:
            cmds = [(0.0, 0.0, 0.0, 0.0), (u_range[0], 0.01, -0.02, 0.005), (-u_range[0], 0.0, 0.0, 0.0)]
            cmds += [tuple((rng.random(4) * 2 - 1) * u_range) for _ in range(2)]
        for c in cmds:
            rows.append((yaw, c))
            if kind == "drone":
                s = np.zeros(12)
                s[0:2] = (rng.random(2) * 2 - 1) * math.radians(30)  # roll, pitch up to +-30 degrees
                s[3:6] = (rng.random(3) * 2 - 1) * 2.0  # p, q, r
                s[6:9] = (rng.random(3) * 2 - 1) * 0.5
                s[11] = rng.random()
                states.append(s)
    u = np.array([c for _, c in rows], dtype=np.float32)
    rot = np.array([y for y, _ in rows], dtype=np.float32)
    ang_vel = ((rng.random(len(rows)) * 2 - 1) * 1.5).astype(np.float32)
    return u, rot, ang_vel, (np.array(states, dtype=np.float32) if states else None)


KIN = {
    # kind: (action size, u_range, agent kwargs, model kwargs)
    "diff": (2, [1.0, 2.0], dict(mass=1.3), dict()),
    "bicycle": (2, [1.0, 1.6], dict(mass=0.9), dict(width=0.08, l_f=0.07, l_r=0.04, max_steering_angle=1.4)),
    "drone": (4, [3.0, 0.1, 0.1, 0.1], dict(mass=0.3), dict(I_xx=8.1e-3, I_yy=9.0e-3, I_zz=14.2e-3)),
}


def make_scenario(agents, dt=0.1):
    """``agents``: [(kind, u_range, u_multiplier, extra)] with kind in holo, holo_rot, diff, bicycle, drone (the last
    three take ``extra = (agent kwargs, model kwargs, integration)``).  No collisions: only the ingest matters."""
    from crafted import _ns

    ns = _ns("vectorizedmultiagentsimulator_b200")
    Agent, World, Sphere = ns["Agent"], ns["World"], ns["Sphere"]

    class IngestCases(ns["BaseScenario"]):
        def make_world(self, batch_dim, device, **kwargs):
            world = World(batch_dim, device, dt=dt, substeps=1)
            for i, (kind, u_range, mult, extra) in enumerate(agents):
                kw = dict(name=f"{kind}_{i}", shape=Sphere(0.05), collide=False, u_range=list(u_range),
                          u_multiplier=list(mult), action_size=len(u_range))
                if kind == "holo":
                    dyn = None
                elif kind == "holo_rot":
                    dyn = ns["HolonomicWithRotation"]()
                    kw["rotatable"] = True
                else:
                    agent_kw, model_kw, integration = extra
                    cls = dict(diff=ns["DiffDrive"], bicycle=ns["KinematicBicycle"], drone=ns["Drone"])[kind]
                    dyn = cls(world, integration=integration, **model_kw)
                    kw.update(rotatable=True, **agent_kw)
                if dyn is not None:
                    kw["dynamics"] = dyn
                world.add_agent(Agent(**kw))
            return world

        def reset_world_at(self, env_index=None):
            pass

        def reward(self, agent):
            return torch.zeros(self.world.batch_dim, device=self.world.device)

        def observation(self, agent):
            return agent.state.pos

    return IngestCases()
