"""``balance``: agents under a bar carry a package to a goal against gravity.

Task definition of the reference's ``vmas/scenarios/balance.py`` (world :17-84, reset :86-213,
reward :220-239, observation :241-257, done :259-263) re-written on the public API for the
CUDA build: same entities, constants, random-draw order, observation layout and reward, but
no host synchronisation in ``reward`` (masked assignment → ``torch.where``) and the three
overlap tests are single kernel launches.
"""
import torch

from ..simulator import observe as O
from ..simulator.program import StepProgram
from ..simulator.core import Agent, Box, Landmark, Line, Sphere, World
from ..simulator.scenario import BaseScenario
from ..simulator.utils import Color, ScenarioUtils


class Scenario(BaseScenario):
    supports_masked_reset = True  # reset_world_at(env_index): None, an int, or a [B] bool mask
    #: observation() reads the world state only (nothing reward() / done() computed): the environment
    #: may run it on a side stream next to the reward callbacks
    observations_are_independent = True

    def make_world(self, batch_dim: int, device: torch.device, **kwargs):
        self._obs_plan = self._obs_all = self._rew_consts = self._package_on_goal = self._program = None
        self.n_agents = kwargs.pop("n_agents", 3)
        self.package_mass = kwargs.pop("package_mass", 5)
        self.random_package_pos_on_line = kwargs.pop("random_package_pos_on_line", True)
        ScenarioUtils.check_kwargs_consumed(kwargs)
        assert self.n_agents > 1

        self.line_length = 0.8
        self.agent_radius = 0.03
        self.shaping_factor = 100
        self.fall_reward = -10
        self.visualize_semidims = False

        world = World(batch_dim, device, gravity=(0.0, -0.05), y_semidim=1)
        for i in range(self.n_agents):
            world.add_agent(
                Agent(name=f"agent_{i}", shape=Sphere(self.agent_radius), u_multiplier=0.7)
            )

        goal = Landmark(name="goal", collide=False, shape=Sphere(), color=Color.LIGHT_GREEN)
        world.add_landmark(goal)
        self.package = Landmark(
            name="package",
            collide=True,
            movable=True,
            shape=Sphere(),
            mass=self.package_mass,
            color=Color.RED,
        )
        self.package.goal = goal
        world.add_landmark(self.package)
        self.line = Landmark(
            name="line",
            shape=Line(length=self.line_length),
            collide=True,
            movable=True,
            rotatable=True,
            mass=5,
            color=Color.BLACK,
        )
        world.add_landmark(self.line)
        self.floor = Landmark(
            name="floor", collide=True, shape=Box(length=10, width=1), color=Color.WHITE
        )
        world.add_landmark(self.floor)

        self.pos_rew = torch.zeros(batch_dim, device=device, dtype=torch.float32)
        self.ground_rew = self.pos_rew.clone()
        return world

    # -- reset ---------------------------------------------------------------------------
    def _uniform(self, n, low, high):
        return torch.zeros((n, 1), device=self.world.device, dtype=torch.float32).uniform_(low, high)

    def _draw(self, env_index, x_bounds, y_bounds):
        """A uniform point per selected env from the device-side stream: ``[B, 2]`` (rows of unselected
        envs are zero), or ``[1, 2]`` for an int ``env_index``."""
        out = self.world.spawn_positions([None], env_index, 0.0, x_bounds, y_bounds, want_positions=True)[:, 0]
        return out[env_index : env_index + 1] if isinstance(env_index, int) else out

    def reset_world_at(self, env_index: int = None):
        world = self.world
        # whatever reward() of the running step cached describes the state before this reset
        self._obs_all, self._obs_from_program, self._done_from_program = None, False, None
        n = 1 if isinstance(env_index, int) else world.batch_dim  # None / bool mask: a row per env
        half = self.line_length / 2
        r_pkg = self.package.shape.radius
        dev = dict(device=world.device, dtype=torch.float32)

        line_y = -world.y_semidim + self.agent_radius * 2
        spread = (-half + r_pkg, half - r_pkg) if self.random_package_pos_on_line else (0.0, 0.0)
        if world.uses_device_reset:
            # CUDA: the three draws come from the respawn kernel's counter-based stream (a uniform point
            # per env; a degenerate y range pins the coordinate), so a masked reset equals one
            # reset_at per env and a shard draws what the unsharded job draws
            goal_pos = self._draw(env_index, (-1.0, 1.0), (0.0, world.y_semidim))
            line_pos = self._draw(env_index, (-1.0 + half, 1.0 - half), (line_y, line_y))
            package_rel = self._draw(env_index, spread, (r_pkg, r_pkg))
        else:
            # draw order matters for seed-for-seed equality with the reference
            goal_pos = torch.cat([self._uniform(n, -1.0, 1.0), self._uniform(n, 0.0, world.y_semidim)], dim=1)
            line_pos = torch.cat([self._uniform(n, -1.0 + half, 1.0 - half), torch.full((n, 1), line_y, **dev)], dim=1)
            package_rel = torch.cat([self._uniform(n, *spread), torch.full((n, 1), r_pkg, **dev)], dim=1)

        offsets, floor_pos = self._reset_constants()
        for i, agent in enumerate(world.agents):
            agent.set_pos(line_pos + offsets[i], batch_index=env_index)

        self.line.set_pos(line_pos, batch_index=env_index)
        self.package.goal.set_pos(goal_pos, batch_index=env_index)
        self.line.set_rot(torch.zeros(1, **dev), batch_index=env_index)
        self.package.set_pos(line_pos + package_rel, batch_index=env_index)
        self.floor.set_pos(floor_pos, batch_index=env_index)
        self.compute_on_the_ground()
        dist = torch.linalg.vector_norm(self.package.state.pos - self.package.goal.state.pos, dim=1)
        self.keep(self, "global_shaping", dist * self.shaping_factor, env_index)

    def _reset_constants(self):
        """Agent offsets under the line ``[A, 2]`` and the floor position ``[2]``, uploaded once per
        device (a ``torch.tensor([...], device=cuda)`` per reset is a synchronous host copy, which
        also cannot be captured in a CUDA graph — ``auto_reset`` in graph mode resets inside one)."""
        world = self.world
        cached = getattr(self, "_reset_consts", None)
        if cached is None or cached[0].device != world.slab.pos.device:
            span = self.line_length - self.agent_radius
            offsets = torch.tensor(
                [[-span / 2 + i * span / (self.n_agents - 1), -self.agent_radius * 2] for i in range(self.n_agents)],
                device=world.device,
                dtype=torch.float32,
            )
            floor_pos = torch.tensor(
                [0, -world.y_semidim - self.floor.shape.width / 2 - self.agent_radius], device=world.device
            )
            cached = self._reset_consts = (offsets, floor_pos)
        return cached

    def compute_on_the_ground(self):
        # the three overlap tests of a step (two here, one in done()) in one launch
        overlaps = self.world.are_overlapping(
            [(self.line, self.floor), (self.package, self.floor), (self.package, self.package.goal)]
        )
        self.on_the_ground = overlaps[0] + overlaps[1]
        self._package_on_goal = overlaps[2]  # consumed by the next done()

    # -- per-step callbacks --------------------------------------------------------------------
    def _step_program(self):
        """reward(), done() and info() of a step as ONE launch (fused with the observation gather): the
        three overlap tests, the shaping term and the glue between them (ref scenarios/balance.py:216-263)."""
        prog = self._program
        if prog is None or prog.world is not self.world:
            p = StepProgram(self.world)
            on_line = p.overlap(self.line, self.floor)
            on_floor = p.overlap(self.package, self.floor)
            on_goal = p.overlap(self.package, self.package.goal)
            on_ground = p.logical_or(on_line, on_floor)
            pos_rew, dist = p.shaping(self.package, self.package.goal, self.shaping_factor, prev=lambda: self.global_shaping)
            ground_rew = p.where(on_ground, p.const(float(self.fall_reward)), p.const(0.0))
            # outputs (fp32 block: shared reward, pos_rew, ground_rew, package distance; bool block: flags)
            p.out_rew = p.store(p.add(ground_rew, pos_rew))
            p.out_pos_rew = p.store(pos_rew)
            p.out_ground_rew = p.store(ground_rew)
            p.out_dist = p.store(dist)
            p.out_on_ground = p.store(on_ground)
            p.out_done = p.store(p.logical_or(on_ground, on_goal))
            prog = self._program = p.finalize()
        return prog

    def reward(self, agent: Agent):
        if agent is self.world.agents[0]:
            prog = self._step_program()
            # the observations of the step ride in the same launch; observation() hands them out
            self._obs_all = prog.run(observe=self._observation_plan())
            self._obs_from_program = True
            self.on_the_ground = prog.out_on_ground.tensor
            self._done_from_program = prog.out_done.tensor
            self.package_dist, self.pos_rew = prog.out_dist.tensor, prog.out_pos_rew.tensor
            self.ground_rew = prog.out_ground_rew.tensor
            self._shared_rew = prog.out_rew.tensor  # the same for every agent
        return self._shared_rew

    def _observation_plan(self):
        plan = getattr(self, "_obs_plan", None)
        if plan is None:
            package, line = self.package, self.line
            plan = self._obs_plan = O.ObservationPlan(
                [
                    [
                        O.pos(a),
                        O.vel(a),
                        O.rel_pos(a, package),
                        O.rel_pos(a, line),
                        O.rel_pos(package, package.goal),
                        O.vel(package),
                        O.vel(line),
                        O.ang_vel(line),
                        O.rot_remainder(line, torch.pi),
                    ]
                    for a in self.world.agents
                ]
            )
        return plan

    def _observe_all(self):
        """Observations of every agent, ``[A, B, 16]``, assembled by one kernel over the state
        slab (same fp32 arithmetic as a per-agent ``torch.cat`` of the nine terms).  Agent-major:
        each agent's ``[B, 16]`` observation is a contiguous slice."""
        return self.world.observe(self._observation_plan())

    def observation(self, agent: Agent):
        agents = self.world.agents
        fresh = getattr(self, "_obs_from_program", False)  # reward() of this step already produced the block
        if (agent is agents[0] and not fresh) or getattr(self, "_obs_all", None) is None:
            self._obs_all = self._observe_all()
        row = self._obs_all[agents.index(agent)]
        if agent is agents[-1]:
            self._obs_all = None  # one sweep over the agents per block: a later call measures anew
            self._obs_from_program = False
        return row

    def done(self):
        from_program, self._done_from_program = getattr(self, "_done_from_program", None), None
        if from_program is not None:  # reward() of this step computed it
            return from_program
        on_goal, self._package_on_goal = getattr(self, "_package_on_goal", None), None
        if on_goal is None:  # no reward() / reset since the last done(): test the current state
            on_goal = self.world.is_overlapping(self.package, self.package.goal)
        return self.on_the_ground + on_goal

    def info(self, agent: Agent):
        return {"pos_rew": self.pos_rew, "ground_rew": self.ground_rew}
