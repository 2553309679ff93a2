"""``transport``: agents push heavy box packages onto a goal.

Task definition of the reference's ``vmas/scenarios/transport.py`` (world :16-67, reset :69-127,
reward :129-166, observation :168-185, done :187-194) re-written on the public API.  Two extra
kwargs build the BASELINE.json variant that the reference does not ship
(``n_lines`` movable/rotatable Line landmarks, ``substeps``); with their defaults the world is
the stock one.
"""
import torch

from ..simulator import observe as O
from ..simulator.core import Agent, Box, Landmark, Line, Sphere, World
from ..simulator.scenario import BaseScenario
from ..simulator.utils import Color, ScenarioUtils


class _Package(Landmark):
    """A package shows red until it sits on its goal, then green (ref transport.py:157-161, set there by
    every reward()); here the colour is derived from the goal flag when somebody asks for it."""

    @property
    def color(self):
        on_goal = getattr(self, "on_goal", None)
        if on_goal is None:
            return Color.RED.value
        red = torch.tensor(Color.RED.value, device=on_goal.device, dtype=torch.float32)
        green = torch.tensor(Color.GREEN.value, device=on_goal.device, dtype=torch.float32)
        return torch.where(on_goal.unsqueeze(-1), green, red)

    @color.setter
    def color(self, color):
        self._color = color


class Scenario(BaseScenario):
    supports_masked_reset = True  # reset_world_at(env_index): None, an int, or a [B] bool mask

    def make_world(self, batch_dim: int, device: torch.device, **kwargs):
        self._obs_plan = self._obs_all = self._shaping_block = self._zero = self._program = None
        n_agents = kwargs.pop("n_agents", 4)
        self.n_packages = kwargs.pop("n_packages", 1)
        self.package_width = kwargs.pop("package_width", 0.15)
        self.package_length = kwargs.pop("package_length", 0.15)
        self.package_mass = kwargs.pop("package_mass", 50)
        self.n_lines = kwargs.pop("n_lines", 0)  # bench.py variant only
        self.line_length = kwargs.pop("line_length", 0.3)
        substeps = kwargs.pop("substeps", 1)
        ScenarioUtils.check_kwargs_consumed(kwargs)

        self.shaping_factor = 100
        self.world_semidim = 1
        self.agent_radius = 0.03

        semidim = self.world_semidim + 2 * self.agent_radius + max(self.package_length, self.package_width)
        world = World(batch_dim, device, x_semidim=semidim, y_semidim=semidim, substeps=substeps)
        for i in range(n_agents):
            world.add_agent(Agent(name=f"agent_{i}", shape=Sphere(self.agent_radius), u_multiplier=0.6))
        goal = Landmark(name="goal", collide=False, shape=Sphere(radius=0.15), color=Color.LIGHT_GREEN)
        world.add_landmark(goal)
        self.packages = []
        for i in range(self.n_packages):
            package = _Package(
                name=f"package {i}",
                collide=True,
                movable=True,
                mass=self.package_mass,
                shape=Box(length=self.package_length, width=self.package_width),
                color=Color.RED,
            )
            package.goal = goal
            self.packages.append(package)
            world.add_landmark(package)
        self.lines = []
        for i in range(self.n_lines):
            line = Landmark(
                name=f"line {i}",
                collide=True,
                movable=True,
                rotatable=True,
                shape=Line(length=self.line_length),
                color=Color.BLACK,
            )
            self.lines.append(line)
            world.add_landmark(line)
        return world

    def reset_world_at(self, env_index: int = None):
        world = self.world
        bounds = (-self.world_semidim, self.world_semidim)
        ScenarioUtils.spawn_entities_randomly(
            world.agents,
            world,
            env_index,
            min_dist_between_entities=self.agent_radius * 2,
            x_bounds=bounds,
            y_bounds=bounds,
        )
        occupied = torch.stack([a.state.pos for a in world.agents], dim=1)
        if isinstance(env_index, int):  # None / bool mask: a row per env
            occupied = occupied[env_index].unsqueeze(0)
        goal = world.landmarks[0]
        ScenarioUtils.spawn_entities_randomly(
            [goal] + self.packages + self.lines,
            world,
            env_index,
            min_dist_between_entities=max(
                p.shape.circumscribed_radius() + goal.shape.radius + 0.01 for p in self.packages
            ),
            x_bounds=bounds,
            y_bounds=bounds,
            occupied_positions=occupied,
        )
        self._obs_all, self._obs_from_program, self._done_from_program = None, False, None
        for package in self.packages:
            dist = torch.linalg.vector_norm(package.state.pos - package.goal.state.pos, dim=1)
            self.keep(package, "global_shaping", dist * self.shaping_factor, env_index)
        prog = self._step_program()
        for k, package in enumerate(self.packages):
            # the goal flags live in the program's outputs (written in place: a captured step keeps their address)
            on_goal = world.is_overlapping(package, package.goal)
            prog.out_on_goal[k].tensor.copy_(on_goal)
            prog.out_on_goal_value[k].tensor.copy_(on_goal)
            package.on_goal = prog.out_on_goal[k].tensor

    def _step_program(self):
        """reward() / done() / the ``on_goal`` observation columns as one step program (ref transport.py:129-194):
        per package the distance-shaping term, the goal test, the reward contribution (0 once on the goal);
        the episode ends when every package is on its goal."""
        prog = getattr(self, "_program", None)
        if prog is not None and prog.world is self.world:
            return prog
        from ..simulator.program import StepProgram

        block = getattr(self, "_shaping_block", None)
        if block is None:  # every package's carried shaping term as one [K, B] block
            for package in self.packages:
                if getattr(package, "global_shaping", None) is None:  # (no reset yet)
                    package.global_shaping = torch.zeros(self.world.batch_dim, device=self.world.device)
            block = self._shaping_block = torch.stack([p.global_shaping for p in self.packages])
            for k, package in enumerate(self.packages):
                package.global_shaping = block[k]
        p = StepProgram(self.world)
        rew, done = p.const(0.0), None
        p.out_dist, p.out_on_goal, p.out_on_goal_value = [], [], []
        for k, package in enumerate(self.packages):
            shaped, dist = p.shaping(package, package.goal, self.shaping_factor, prev=lambda k=k: self._shaping_block[k])
            on_goal = p.overlap(package, package.goal)
            rew = p.add(rew, p.where(on_goal, p.const(0.0), shaped))
            done = on_goal if done is None else p.logical_and(done, on_goal)
            p.out_dist.append(p.store(dist))
            p.out_on_goal.append(p.store(on_goal))
            p.out_on_goal_value.append(p.store(on_goal, torch.float32))  # the observation column (0. / 1.)
        p.out_rew, p.out_done = p.store(rew), p.store(done, torch.bool)
        self._program = p.finalize()
        return self._program

    def _observation_plan(self):
        plan = getattr(self, "_obs_plan", None)
        if plan is None:
            prog = self._step_program()
            plan = self._obs_plan = O.ObservationPlan(
                [
                    [O.pos(a), O.vel(a)]
                    + [
                        t
                        for package, flag in zip(self.packages, prog.out_on_goal_value)
                        for t in (O.rel_pos(package, package.goal), O.rel_pos(package, a), O.vel(package), O.value(flag))
                    ]
                    for a in self.world.agents
                ]
            )
        return plan

    def reward(self, agent: Agent):
        if agent is self.world.agents[0]:
            prog = self._step_program()
            # one launch (captured: the epilogue of the step's kernel) for the reward, the flags and the
            # observations of the step; observation() hands the block out
            self._obs_all = prog.run(observe=self._observation_plan())
            self._obs_from_program = True
            for k, package in enumerate(self.packages):
                package.dist_to_goal = prog.out_dist[k].tensor
                package.on_goal = prog.out_on_goal[k].tensor
            self.rew = prog.out_rew.tensor
            self._done_from_program = prog.out_done.tensor
        return self.rew

    def observation(self, agent: Agent):
        agents = self.world.agents
        fresh = getattr(self, "_obs_from_program", False)  # reward() of this step already produced the block
        if (agent is agents[0] and not fresh) or getattr(self, "_obs_all", None) is None:
            # (after a reset: the goal flags of the program's outputs were refreshed there)
            self._obs_all = self.world.observe(self._observation_plan())
        row = self._obs_all[agents.index(agent)]
        if agent is agents[-1]:
            self._obs_all = None  # one sweep over the agents per block: a later call measures anew
            self._obs_from_program = False
        return row

    def done(self):
        from_program, self._done_from_program = getattr(self, "_done_from_program", None), None
        if from_program is not None:  # reward() of this step computed it
            return from_program
        return torch.stack([p.on_goal for p in self.packages], dim=1).all(dim=-1)
