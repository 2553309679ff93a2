"""A crafted world with per-env physical parameters (domain randomisation) (TEST INFRASTRUCTURE).

``randomised``: sphere, box and line entities in contact and one joint; per-env ``[B, 1]`` masses on
holonomic agents and on a landmark, per-env linear and angular friction coefficients, per-env gravity on
one entity, world gravity and friction, ``max_f`` on one agent.  The values are drawn at every reset and
half the envs are re-drawn every ``REDRAW_EVERY`` steps in ``pre_step`` — alternately by in-place edits of
the entities' tensors and by assigning fresh tensors (angular friction: in place only, the reference's
``Entity.angular_friction`` has no setter; its tensors come from the constructors).

Like ``tests/crafted.py`` the scenario is built from whichever namespace it is given: the UNMODIFIED
reference's ``vmas`` (``tests/make_golden_params.py`` records its roll-out) or this package's.
"""
import math

import torch

from crafted import _ns, _scatter

REDRAW_EVERY = 3
#: entity name -> the attributes it holds per env (gravity: a [B, 2] tensor)
PER_ENV = {
    "agent_0": ("mass", "linear_friction", "angular_friction"),
    "agent_1": ("mass",),
    "agent_2": ("linear_friction", "gravity"),
    "crate": ("mass", "angular_friction"),
    "disc": ("mass",),
}
#: [low, high) of each attribute's draw
RANGES = {"mass": (0.5, 3.0), "linear_friction": (0.02, 0.3), "angular_friction": (0.01, 0.2), "gravity": (-0.3, 0.3)}


def per_env_values(world):
    """{entity index: {attribute: [B, k] tensor}} of the per-env attributes, as ``World.step`` reads them now."""
    out = {}
    for i, e in enumerate(world.entities):
        attrs = PER_ENV.get(e.name)
        if attrs:
            out[i] = {a: getattr(e, a).clone() for a in attrs}
    return out


def make_scenario(root, seed=4321):
    ns = _ns(root)
    Agent, Landmark, World = ns["Agent"], ns["Landmark"], ns["World"]
    Sphere, Box, Line, Joint = ns["Sphere"], ns["Box"], ns["Line"], ns["Joint"]
    Rot = ns["HolonomicWithRotation"]

    class Randomised(ns["BaseScenario"]):
        def make_world(self, batch_dim, device, **kwargs):
            self.gen = torch.Generator().manual_seed(seed)
            self.t = 0
            world = World(
                batch_dim, device, substeps=3, drag=0.2, linear_friction=0.05, gravity=(0.0, -0.1),
                joint_force=6, x_semidim=0.5, y_semidim=0.5,
            )
            ones = torch.ones(batch_dim, 1, device=device)
            world.add_agent(Agent(name="agent_0", shape=Sphere(0.06), rotatable=True, dynamics=Rot(), max_f=0.8,
                                  u_multiplier=[1.0, 1.0, 0.02], mass=ones.clone(), linear_friction=0.1 * ones,
                                  angular_friction=0.05 * ones))
            world.add_agent(Agent(name="agent_1", shape=Box(0.14, 0.08), rotatable=True, dynamics=Rot(),
                                  u_multiplier=[1.0, 1.0, 0.02], angular_friction=0.1))
            world.add_agent(Agent(name="agent_2", shape=Line(0.25), rotatable=True, dynamics=Rot(),
                                  u_multiplier=[1.0, 1.0, 0.02], mass=1.5))
            world.add_landmark(Landmark("crate", shape=Box(0.15, 0.12), movable=True, rotatable=True, collide=True,
                                        angular_friction=0.05 * ones))
            world.add_landmark(Landmark("disc", shape=Sphere(0.08), movable=True, collide=True,
                                        linear_friction=0.2))
            world.add_joint(Joint(world.agents[0], world.agents[1], anchor_a=(0, 0), anchor_b=(-1, 0), dist=0.2,
                                  rotate_a=True, rotate_b=True, collidable=False, width=0, mass=1))
            self.spread = 0.25
            return world

        def _draw(self, n, attr):
            lo, hi = RANGES[attr]
            k = 2 if attr == "gravity" else 1
            return torch.rand(n, k, generator=self.gen) * (hi - lo) + lo

        def _set_params(self, envs, in_place):
            """New values for the envs ``envs`` (a [B] bool mask): in place, or by assigning a fresh tensor."""
            world = self.world
            n = world.batch_dim
            for e in world.entities:
                for attr in PER_ENV.get(e.name, ()):
                    new = self._draw(n, attr).to(world.device)
                    cur = getattr(e, attr)
                    if not isinstance(cur, torch.Tensor) or cur.dim() != 2:
                        setattr(e, attr, new)  # (the first reset: from the constructor's scalar)
                    elif in_place or attr == "angular_friction":  # (the reference has no angular_friction setter)
                        cur[envs] = new[envs]
                    else:
                        setattr(e, attr, torch.where(envs.unsqueeze(-1), new, cur))

        def reset_world_at(self, env_index=None):
            world = self.world
            n = world.batch_dim
            _scatter(world, world.entities, self.gen, self.spread, env_index, math.pi / 2)
            for e in world.entities:
                if e.movable:
                    v = (torch.rand(n, 2, generator=self.gen) * 2 - 1) * 0.3
                    e.set_vel(v.to(world.device) if env_index is None else v[env_index].to(world.device),
                              batch_index=env_index)
                if e.rotatable:
                    w = (torch.rand(n, 1, generator=self.gen) * 2 - 1) * 1.0
                    e.set_ang_vel(w.to(world.device) if env_index is None else w[env_index].to(world.device),
                                  batch_index=env_index)
            envs = torch.zeros(n, dtype=torch.bool, device=world.device)
            envs[slice(None) if env_index is None else env_index] = True
            self._set_params(envs, in_place=self.t > 0)

        def pre_step(self):
            self.t += 1
            if self.t % REDRAW_EVERY == 0:  # half the envs, alternately in place and by re-assignment
                n = self.world.batch_dim
                envs = (torch.arange(n) % 2 == (self.t // REDRAW_EVERY) % 2).to(self.world.device)
                self._set_params(envs, in_place=(self.t // REDRAW_EVERY) % 2 == 0)

        def reward(self, agent):
            return torch.zeros(self.world.batch_dim, device=self.world.device)

        def observation(self, agent):
            return torch.cat([agent.state.pos, agent.state.vel], dim=-1)

    return Randomised()
