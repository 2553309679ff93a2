"""The captured step of a scenario whose observations read LIDARs, as ONE launch: ``step_env_kernel`` casts the rays in
its epilogue (``spec_lidar``) and writes the readings into the observation rows.  It must return, bit for bit, what the
eager step, the two-launch step (ingest kernel, then the whole-step kernel; ``_INGEST_IN_KERNEL = False``) and the
graph replay (``_DIRECT_STEP = False``, where ``cast_rays_batched_kernel`` casts them) return — observations, rewards,
dones and the physics state — over several steps with ``reset_at(dones)`` between them.

Two scenarios written on a ``StepProgram`` and an ``ObservationPlan``, defined here:

* ``LidarNavigation``: navigation's world (sphere agents whose LIDARs see the other agents, 2 substeps) with a shaping
  and on-goal reward as a program, without the batch-wide ``collides`` gate.  No masked pairs: no grid barrier.
* ``LidarBalance``: balance with a LIDAR on every agent that sees the other agents, the package, the line and the box
  floor.  Line and box pairs are masked: the kernel runs the grid barrier.

Also covered: ``range_minus_distance`` both ways, fp16 and bf16 observations, a batch past what the GPU holds at once,
a sensor with more targets than the epilogue takes (it stays on the graph route), ``max_steps`` with LIDARs, and
``Lidar._last_measurement`` on the one-kernel step.
"""
import gc

import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from vectorizedmultiagentsimulator_b200 import _native, codegen
from vectorizedmultiagentsimulator_b200.scenarios import balance, navigation
from vectorizedmultiagentsimulator_b200.simulator import observe as O
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E
from vectorizedmultiagentsimulator_b200.simulator.program import StepProgram
from vectorizedmultiagentsimulator_b200.simulator.sensors import Lidar

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
SLAB = ("pos", "vel", "rot", "ang_vel", "force", "torque")


class LidarNavigation(navigation.Scenario):
    """Navigation's world and reset; reward, dones and observations as one program + observation launch."""

    def make_world(self, batch_dim, device, **kwargs):
        self.range_minus_distance = kwargs.pop("range_minus_distance", True)
        self._prog = self._plan = self._obs = self._dones = None
        return super().make_world(batch_dim, device, **kwargs)

    def _program(self):
        if self._prog is None or self._prog.world is not self.world:
            p = StepProgram(self.world)
            total = reached = None
            for a in self.world.agents:
                rew, dist = p.shaping(a, a.goal, self.pos_shaping_factor, prev=lambda a=a: a.pos_shaping)
                on_goal = p.lt(dist, p.const(float(a.goal.shape.radius)))
                total = rew if total is None else p.add(total, rew)
                reached = on_goal if reached is None else p.logical_and(reached, on_goal)
            final = p.where(reached, p.const(float(self.final_reward)), p.const(0.0))
            p.out_rew = p.store(p.add(total, final))
            p.out_done = p.store(reached)
            self._prog = p.finalize()
        return self._prog

    def _observation_plan(self):
        if self._plan is None:
            self._plan = O.ObservationPlan(
                [[O.pos(a), O.vel(a), O.rel_pos(a, a.goal), O.lidar(a.sensors[0], self.range_minus_distance)]
                 for a in self.world.agents]
            )
        return self._plan

    def reward(self, agent):
        if agent is self.world.agents[0]:
            prog = self._program()
            self._obs = prog.run(observe=self._observation_plan())
            self._rew, self._dones = prog.out_rew.tensor, prog.out_done.tensor
        return self._rew

    def observation(self, agent):
        agents = self.world.agents
        if self._obs is None:
            self._obs = self.world.observe(self._observation_plan())
        row = self._obs[agents.index(agent)]
        if agent is agents[-1]:
            self._obs = None
        return row

    def done(self):
        dones, self._dones = self._dones, None
        if dones is None:
            dones = torch.stack([torch.linalg.vector_norm(a.state.pos - a.goal.state.pos, dim=-1) < a.goal.shape.radius
                                 for a in self.world.agents]).all(0)
        return dones

    def info(self, agent):
        return {}


class LidarBalance(balance.Scenario):
    """Balance with a LIDAR on every agent: it sees the other agents, the package, the line and the floor."""

    def make_world(self, batch_dim, device, **kwargs):
        self.range_minus_distance = kwargs.pop("range_minus_distance", False)
        n_rays = kwargs.pop("n_rays", 7)
        world = super().make_world(batch_dim, device, **kwargs)
        for a in world.agents:
            a.add_sensor(Lidar(world, n_rays=n_rays, max_range=0.6, entity_filter=lambda e: e.collide))
        return world

    def _observation_plan(self):
        plan = getattr(self, "_obs_plan", None)
        if plan is None:
            plan = super()._observation_plan()
            self._obs_plan = plan = O.ObservationPlan(
                [row + [O.lidar(a.sensors[0], self.range_minus_distance)] for row, a in zip(plan.rows, self.world.agents)]
            )
        return plan


def _actions(env, gen):
    out = []
    for agent in env.agents:
        r = agent.action.u_range_tensor.cpu()
        out.append(((torch.rand(env.num_envs, agent.action_size, generator=gen) * 2 - 1) * r).cuda())
    return out


def _make(cls, kwargs, n, monkeypatch, flags=None, cuda_graph=True, **env_kw):
    with monkeypatch.context() as m:
        for k, v in (flags or {}).items():
            m.setattr(E, k, v)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)  # (the LIDAR table is part of the kernel: compiled at capture)
        env = b200.make_env(cls(), num_envs=n, device="cuda", seed=0, cuda_graph=cuda_graph, **env_kw, **kwargs)
        env.reset()
        if cuda_graph:  # (the flags are read when the step is captured: warm-up steps + capture happen here)
            gen = torch.Generator().manual_seed(1)
            for _ in range(4):
                env.step(_actions(env, gen))
    return env


def _same(g, w):
    return torch.equal(g, w) if EXACT else same_result(g.float(), w.float(), atol=2e-4)


def _check(got, want, env, ref, what):
    for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
        assert g.dtype == w.dtype and g.shape == w.shape and _same(g, w), f"{what}: output leaf {i}"
    assert torch.equal(env.steps, ref.steps), f"{what}: steps"
    for k in SLAB:
        assert _same(getattr(env.world.slab, k), getattr(ref.world.slab, k)), f"{what}: slab {k}"


def _variants(cls, kwargs, n, monkeypatch, two_launches=True, graph=True, **env_kw):
    gc.collect()  # (the envs of earlier tests go now, not in the middle of a capture below)
    torch.cuda.synchronize()
    envs = {
        "eager": _make(cls, kwargs, n, monkeypatch, cuda_graph=False, **env_kw),
        "one kernel": _make(cls, kwargs, n, monkeypatch, **env_kw),
    }
    if two_launches:
        envs["two launches"] = _make(cls, kwargs, n, monkeypatch, dict(_INGEST_IN_KERNEL=False), **env_kw)
    if graph:
        envs["graph"] = _make(cls, kwargs, n, monkeypatch, dict(_DIRECT_STEP=False), **env_kw)
    ref = envs["eager"]
    for env in envs.values():
        if env is not ref:
            sync_env(ref, env)
    return envs


def _assert_one_kernel(env):
    plan = env._one_call
    assert plan is not None and plan.direct and plan.c.ingest_in_kernel == 1 and plan.c.fused_kernel > 0


def _run(envs, steps=6, reset_dones=True):
    """Steps every env with the same actions ("eager" is the reference); one launch per step on "one kernel";
    ``reset_at(dones)`` after every step."""
    ref, one = envs["eager"], envs.get("one kernel")
    gen = torch.Generator().manual_seed(7)
    for t in range(steps):
        actions = _actions(ref, gen)
        want = ref.step([a.clone() for a in actions])
        for label, env in envs.items():
            if env is ref:
                continue
            backend = env.world._get_backend()
            before = backend.launches
            got = env.step([a.clone() for a in actions])
            if env is one:
                assert backend.launches - before == 1, f"{label} step {t}: {backend.launches - before} launches"
            _check(got, want, env, ref, f"{label} step {t}")
            if not EXACT:
                sync_env(ref, env)
        if reset_dones:
            dones = want[2]
            want_obs = ref.reset_at(dones)
            for label, env in envs.items():
                if env is not ref:
                    for i, (g, w) in enumerate(zip(flatten(env.reset_at(dones)), flatten(want_obs))):
                        assert _same(g, w), f"{label} reset_at obs {i}"
                    sync_env(ref, env)
    return want


CASES = [
    (LidarNavigation, dict(n_agents=4, range_minus_distance=True)),
    (LidarNavigation, dict(n_agents=4, range_minus_distance=False)),
    (LidarBalance, dict(n_agents=4, range_minus_distance=False)),
    (LidarBalance, dict(n_agents=3, range_minus_distance=True)),
]


def _id(case):
    cls, kwargs = case
    return f"{cls.__name__}-{'-'.join(f'{k}{v}' for k, v in kwargs.items())}"


@pytest.mark.parametrize("cls,kwargs", CASES, ids=[_id(c) for c in CASES])
def test_one_kernel_step_equals_eager_two_launches_and_graph(cls, kwargs, monkeypatch):
    envs = _variants(cls, kwargs, 1001, monkeypatch)  # 1001 envs: lane pairs (G = 2)
    _assert_one_kernel(envs["one kernel"])
    assert envs["two launches"]._one_call.c.ingest_in_kernel == 0 and envs["two launches"]._one_call.c.fused_kernel > 0
    assert envs["graph"]._one_call is None or not envs["graph"]._one_call.direct
    want = _run(envs)
    # the readings are not all max_range: the rays hit something
    ref = envs["eager"]
    plan = ref.scenario._observation_plan()
    r, c, sensor, flipped = plan.compile(ref.world)[1][0]
    readings = want[0][r][:, c : c + sensor._angles.shape[1]]
    far = 0.0 if flipped else float(sensor._max_range)
    assert (readings != far).any()


@pytest.mark.parametrize("cls,kwargs", [CASES[0], CASES[2]], ids=[_id(CASES[0]), _id(CASES[2])])
def test_last_measurement_views_the_readings(cls, kwargs, monkeypatch):
    envs = _variants(cls, dict(kwargs, range_minus_distance=False), 1001, monkeypatch, two_launches=False)
    _run(envs, steps=2, reset_dones=False)
    got, want = envs["one kernel"], envs["graph"]
    for s_got, s_want in zip((a.sensors[0] for a in got.agents), (a.sensors[0] for a in want.agents)):
        assert s_got._last_measurement is not None and torch.equal(s_got._last_measurement, s_want._last_measurement)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cls,kwargs", [CASES[0], CASES[3]], ids=[_id(CASES[0]), _id(CASES[3])])
def test_sixteen_bit_observations(cls, kwargs, dtype, monkeypatch):
    envs = _variants(cls, kwargs, 1001, monkeypatch, two_launches=False, obs_dtype=dtype)
    _assert_one_kernel(envs["one kernel"])
    _run(envs, steps=4)
    want = _run(envs, steps=1, reset_dones=False)
    assert want[0][0].dtype == dtype
    # no fp32 copy of the readings on the one-kernel step: no measurement view there (INTEGRATION.md)
    assert all(a.sensors[0]._last_measurement is None for a in envs["one kernel"].agents)


def test_batches_on_each_lane_mapping_and_past_the_gpu(monkeypatch):
    """LidarBalance has a grid barrier: lane pairs while the blocks fit the GPU twice over, one lane per env up to
    what fits once, then the ingest launch in front of the whole-step kernel (its epilogue casts the rays too)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cls, kwargs = CASES[2]
    for n, launches in ((sms * 8 * 64 // 2 + 64, 1), (sms * 8 * 64 + 64 * 16, 2)):
        envs = _variants(cls, kwargs, n, monkeypatch, two_launches=False, graph=False)
        _assert_one_kernel(envs["one kernel"])
        one, ref = envs["one kernel"], envs["eager"]
        backend = one.world._get_backend()
        gen = torch.Generator().manual_seed(3)
        for t in range(3):
            actions = _actions(one, gen)
            want = ref.step([a.clone() for a in actions])
            before = backend.launches
            got = one.step([a.clone() for a in actions])
            assert (backend.launches - before == 1) == (launches == 1), f"{n} envs step {t}"
            _check(got, want, one, ref, f"{n} envs step {t}")
        del envs


def test_more_targets_than_the_epilogue_takes_stays_on_the_graph(monkeypatch):
    # 18 agents: each LIDAR sees 17 agents, the package, the line and the floor
    kwargs = dict(n_agents=18, n_rays=4)
    envs = _variants(LidarBalance, kwargs, 257, monkeypatch, two_launches=False)
    ref = envs["eager"]
    sensor = ref.agents[0].sensors[0]
    targets = ref.world._get_backend().ray_targets(sensor.agent, sensor.entity_filter)
    assert len(targets) > codegen.MAX_LIDAR_TARGETS
    for label in ("one kernel", "graph"):
        plan = envs[label]._one_call
        assert plan is None or not plan.direct, label
    del envs["one kernel"]  # (the graph route: compared once)
    _run(envs, steps=3)


def test_max_steps_with_lidars(monkeypatch):
    cls, kwargs = CASES[0]
    envs = _variants(cls, kwargs, 1001, monkeypatch, two_launches=False, max_steps=3)
    _assert_one_kernel(envs["one kernel"])
    ref = envs["eager"]
    ref.steps.copy_((torch.arange(ref.num_envs, dtype=torch.float32) % 3).cuda())
    for env in envs.values():
        if env is not ref:
            sync_env(ref, env)
    _run(envs, steps=5)
