"""Crafted worlds past the thread-per-env step's shared-memory limit (TEST INFRASTRUCTURE).

``large_160``: 160 entities, just past the ~139 a one-thread-per-env layout holds.  Spheres, boxes and
lines; 60 of them collide (1 696 work items, 1 492 of them subject to the batch-wide broad phase: 47 mask
words), scattered densely enough that a few are in contact in every env; two joints with their anchors apart
(one rotating, one at a fixed angle; each joint is two constraints through a landmark of its own); world
gravity, friction, semidims and an agent force clamp.
``large_520``: 520 entities, past the ~500 the observation staging held in 48 KB.
``large_1024``: 1024 entities, the CUDA backend's limit.
The two larger worlds have the same 60 colliding entities and joints; the rest are non-colliding bodies that
only drift and feel friction, so the reference can record them in seconds.

Like ``tests/crafted.py`` the scenario is built from whichever namespace it is given: the UNMODIFIED
reference's ``vmas`` (``tests/make_golden_large.py`` records its roll-outs) or this package's.
"""
import math

import torch

from crafted import _ns, _scatter

N_AGENTS = 8
N_COLLIDING = 60  # agents included


def make_scenario(root, kind, seed=2468):
    """``kind``: ``large_<n>`` — a world of n >= 70 entities (the fixtures: 160, 520, 1024)."""
    ns = _ns(root)
    Agent, Landmark, World = ns["Agent"], ns["Landmark"], ns["World"]
    Sphere, Box, Line, Joint = ns["Sphere"], ns["Box"], ns["Line"], ns["Joint"]
    Rot = ns["HolonomicWithRotation"]
    n_entities = int(kind.split("_")[1])
    assert n_entities >= 70, kind

    def shape(i):
        return (Sphere(0.03), Box(0.07, 0.04), Line(0.09))[i % 3]

    class Large(ns["BaseScenario"]):
        def make_world(self, batch_dim, device, **kwargs):
            self.gen = torch.Generator().manual_seed(seed)
            world = World(
                batch_dim, device, substeps=2, drag=0.2, linear_friction=0.05, gravity=(0.0, -0.05),
                joint_force=6, torque_constraint_force=0.02, x_semidim=1.0, y_semidim=1.0,
            )
            for i in range(N_AGENTS):
                world.add_agent(Agent(name=f"agent_{i}", shape=shape(i), rotatable=True, dynamics=Rot(),
                                      u_multiplier=[1.0, 1.0, 0.02], max_f=0.8 if i == 0 else None))
            for i in range(N_COLLIDING - N_AGENTS):
                movable = i % 4 != 3  # a few static obstacles among them
                world.add_landmark(Landmark(f"obstacle_{i}", shape=shape(i), collide=True, movable=movable,
                                            rotatable=movable, mass=1.5))
            for i in range(n_entities - N_COLLIDING - 2):  # (each joint adds a landmark of its own)
                world.add_landmark(Landmark(f"drifter_{i}", shape=Sphere(0.02), collide=False, movable=i % 2 == 0,
                                            rotatable=i % 4 == 0))
            a = world.agents
            world.add_joint(Joint(a[0], a[1], anchor_a=(0, 0), anchor_b=(-1, 0), dist=0.2, rotate_a=True,
                                  rotate_b=True, collidable=False, width=0, mass=1))
            world.add_joint(Joint(a[2], a[3], anchor_a=(1, 0), anchor_b=(0, 0), dist=0.15, rotate_a=False,
                                  rotate_b=False, fixed_rotation_a=0.3, fixed_rotation_b=0.3, collidable=False,
                                  width=0, mass=1))
            return world

        def reset_world_at(self, env_index=None):
            world = self.world
            n = world.batch_dim
            # the colliding bodies packed into a small square (contacts), the drifters spread out; the jointed
            # agents and the joints' own landmarks at modest angles (a fixed-angle joint's torque grows like
            # exp(|angle difference|) and throws bodies to infinity when started half a turn apart)
            jointed = world.agents[:4] + [e for e in world.landmarks if e.name.startswith("joint ")]
            colliding = [e for e in world.entities if e.collide and e not in jointed]
            drifters = [e for e in world.entities if e not in jointed and e not in colliding]
            _scatter(world, jointed, self.gen, 0.45, env_index, 0.1)
            _scatter(world, colliding, self.gen, 0.45, env_index, math.pi)
            _scatter(world, drifters, self.gen, 0.95, env_index, math.pi)
            for e in world.entities:
                if e.movable:
                    v = (torch.rand(n, 2, generator=self.gen) * 2 - 1) * 0.3
                    e.set_vel(v.to(world.device) if env_index is None else v[env_index].to(world.device),
                              batch_index=env_index)
                if e.rotatable:
                    w = (torch.rand(n, 1, generator=self.gen) * 2 - 1) * (0.1 if e in jointed else 1.0)
                    e.set_ang_vel(w.to(world.device) if env_index is None else w[env_index].to(world.device),
                                  batch_index=env_index)

        def reward(self, agent):
            return torch.zeros(self.world.batch_dim, device=self.world.device)

        def observation(self, agent):
            return torch.cat([agent.state.pos, agent.state.vel], dim=-1)

    return Large()
