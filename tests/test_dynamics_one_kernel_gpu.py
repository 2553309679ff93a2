"""The captured step of scenarios whose agents use other action models (holonomic with rotation, forward, rotation,
differential drive, and worlds that mix them with holonomic agents on a lane pair) as ONE launch:
``step_env_kernel`` whose prologue runs each agent's model.  It must return, bit for bit, what the eager step and the
two-launch captured step (ingest kernel, then the whole-step kernel; ``_INGEST_IN_KERNEL = False``) return —
observations, rewards, dones, infos, the physics state and ``agent.action.u`` — and flag the same illegal actions.

Covered: balance with 3 and 4 agents (a lone agent on a lane pair), transport with 2 lines and 3 substeps (the
batch-wide broad phase behind a grid barrier), continuous, discrete and multi-discrete actions, batches on each lane
mapping and past what the GPU holds at once (two launches again, same bits), 16-bit observations, and a world with a
kinematic bicycle, which stays on two launches.
"""
from types import SimpleNamespace

import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.scenarios import balance, transport
from vectorizedmultiagentsimulator_b200.simulator.dynamics.basic import (
    Forward, Holonomic, HolonomicWithRotation, Rotation,
)
from vectorizedmultiagentsimulator_b200.simulator.dynamics.diff_drive import DiffDrive
from vectorizedmultiagentsimulator_b200.simulator.dynamics.kinematic_bicycle import KinematicBicycle
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
SLAB = ("pos", "vel", "rot", "ang_vel", "force", "torque")
MODEL_DT = SimpleNamespace(dt=0.1)  # (what the kinematic models read of their world)

# name: (dynamics factory, u_range)
MODELS = {
    "holo": (Holonomic, [1.0, 1.0]),
    "holo_rot": (HolonomicWithRotation, [1.0, 0.8, 0.5]),
    "forward": (Forward, [1.2]),
    "rotation": (Rotation, [0.6]),
    "diff": (lambda: DiffDrive(MODEL_DT, integration="rk4"), [1.0, 1.5]),
    "diff_euler": (lambda: DiffDrive(MODEL_DT, integration="euler"), [0.8, 1.0]),
    "bicycle": (lambda: KinematicBicycle(MODEL_DT, width=0.05, l_f=0.06, l_r=0.04, max_steering_angle=0.6), [1.0, 0.8]),
}


def _with_models(base, module, lineup):
    """``base`` (balance or transport) whose agents get the action models of ``lineup`` in turn (rotatable)."""

    class Scenario(base):
        def make_world(self, batch_dim, device, **kwargs):
            orig, count = module.Agent, iter(range(1 << 20))

            def agent(**kw):
                factory, u_range = MODELS[lineup[next(count) % len(lineup)]]
                kw.update(dynamics=factory(), u_range=u_range, rotatable=True)
                return orig(**kw)

            module.Agent = agent
            try:
                return super().make_world(batch_dim, device, **kwargs)
            finally:
                module.Agent = orig

    Scenario.__name__ = f"{base.__module__.rsplit('.', 1)[-1]}[{','.join(lineup)}]"
    return Scenario


def _actions(env, gen, bad=None):
    """Random legal actions per agent (continuous [B, size] fp32; discrete [B, 1] / [B, size] int64) on the device;
    ``bad``: (agent, env, value) written over one of them."""
    out = []
    for agent in env.agents:
        size = agent.action_size
        if env.continuous_actions:
            r = torch.tensor(agent.action.u_range_tensor.tolist())
            a = (torch.rand(env.num_envs, size, generator=gen) * 2 - 1) * r
        elif env.multidiscrete_actions:
            a = torch.stack([torch.randint(0, n, (env.num_envs,), generator=gen) for n in agent.discrete_action_nvec], -1)
        else:
            total = 1
            for n in agent.discrete_action_nvec:
                total *= n
            a = torch.randint(0, total, (env.num_envs, 1), generator=gen)
        out.append(a)
    if bad is not None:
        i, e, v = bad
        out[i][e, -1] = v
    return [a.cuda() for a in out]


def _make(scenario, kwargs, n, monkeypatch, space, flags=None, cuda_graph=True, **env_kw):
    with monkeypatch.context() as m:
        for k, v in (flags or {}).items():
            m.setattr(E, k, v)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)  # (these prologues compile when the step is captured)
        env = b200.make_env(scenario(), num_envs=n, device="cuda", seed=0, continuous_actions=space == "continuous",
                            multidiscrete_actions=space == "multidiscrete", cuda_graph=cuda_graph, **env_kw, **kwargs)
        env.reset()
        if cuda_graph:  # (the flags are read when the step is captured: warm-up steps + capture happen here)
            gen = torch.Generator().manual_seed(1)
            for _ in range(4):
                env.step(_actions(env, gen))
    return env


def _same(g, w):
    """Bit-equal (exact build; NaN where the other has NaN: a NaN action leaves NaN in the state) or within the
    parity tolerance (fast build)."""
    if not EXACT:
        return same_result(g.float(), w.float(), atol=2e-4)
    if g.shape != w.shape or g.dtype != w.dtype:
        return False
    if not g.is_floating_point():
        return torch.equal(g, w)
    return bool(((g == w) | (g.isnan() & w.isnan())).all())


def _check(got, want, env, ref, what):
    for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
        assert g.dtype == w.dtype and _same(g, w), f"{what}: output leaf {i}"
    for k in SLAB:
        assert _same(getattr(env.world.slab, k), getattr(ref.world.slab, k)), f"{what}: slab {k}"
    for a, b in zip(env.agents, ref.agents):
        assert _same(a.action.u, b.action.u), f"{what}: {a.name} action.u"


def _run(envs, steps=10, reset_at=5, bad_at=None):
    """Steps every env with the same actions; the first is the reference.  ``bad_at``: (step, (agent, env, value))."""
    ref, *others = envs.values()
    for env in others:
        sync_env(ref, env)
    gen = torch.Generator().manual_seed(7)
    one = envs.get("one kernel")
    for t in range(steps):
        bad = bad_at[1] if bad_at is not None and bad_at[0] == t else None
        actions = _actions(ref, gen, bad)
        want = ref.step([a.clone() for a in actions])
        for label, env in envs.items():
            if env is ref:
                continue
            backend = env.world._get_backend()
            before = backend.launches
            got = env.step([a.clone() for a in actions])
            if env is one and one._one_call is not None and one._one_call.c.ingest_in_kernel:
                assert backend.launches - before == 1, f"{label} step {t}: {backend.launches - before} launches"
            _check(got, want, env, ref, f"{label} step {t}")
            if not EXACT:
                sync_env(ref, env)
        if bad is not None:
            for label, env in envs.items():
                with pytest.raises(AssertionError):
                    env.check_actions_now()
                env.check_actions_now()  # (the flag was cleared by the raise)
        if t == reset_at:
            want_obs = ref.reset_at(3)
            for label, env in envs.items():
                if env is ref:
                    continue
                got_obs = env.reset_at(3)
                for i, (g, w) in enumerate(zip(flatten(got_obs), flatten(want_obs))):
                    assert _same(g, w), f"{label} reset_at obs {i}"
                sync_env(ref, env)


def _variants(scenario, kwargs, n, monkeypatch, space, two_launches=True, **env_kw):
    envs = {
        "eager": _make(scenario, kwargs, n, monkeypatch, space, cuda_graph=False, **env_kw),
        "one kernel": _make(scenario, kwargs, n, monkeypatch, space, **env_kw),
    }
    if two_launches:
        envs["two launches"] = _make(scenario, kwargs, n, monkeypatch, space, dict(_INGEST_IN_KERNEL=False), **env_kw)
    return envs


def _assert_one_kernel(env):
    plan = env._one_call
    assert plan is not None and plan.c.ingest_in_kernel == 1 and plan.c.fused_kernel > 0


BALANCE3 = _with_models(balance.Scenario, balance, ["holo_rot", "forward", "rotation"])
BALANCE4 = _with_models(balance.Scenario, balance, ["diff", "rotation", "holo", "diff_euler"])
TRANSPORT = _with_models(transport.Scenario, transport, ["holo_rot", "diff", "rotation", "forward"])
CASES = [
    ("balance3", BALANCE3, dict(n_agents=3)),
    ("balance4", BALANCE4, dict(n_agents=4)),
    ("transport3", TRANSPORT, dict(n_agents=4, n_lines=2, substeps=3)),
]


@pytest.mark.parametrize("space", ["continuous", "discrete", "multidiscrete"])
@pytest.mark.parametrize("name,scenario,kwargs", CASES, ids=[c[0] for c in CASES])
def test_one_kernel_step_equals_eager_and_two_launches(name, scenario, kwargs, space, monkeypatch):
    envs = _variants(scenario, kwargs, 1001, monkeypatch, space)  # 1001 envs: lane pairs (G = 2)
    _assert_one_kernel(envs["one kernel"])
    assert envs["two launches"]._one_call.c.ingest_in_kernel == 0
    _run(envs)


@pytest.mark.parametrize("model", ["holo_rot", "forward", "rotation", "diff"])
def test_each_model_alone(model, monkeypatch):
    envs = _variants(_with_models(balance.Scenario, balance, [model]), dict(n_agents=4), 333, monkeypatch, "continuous")
    _assert_one_kernel(envs["one kernel"])
    _run(envs, steps=6, reset_at=3)


def test_illegal_actions_decode_like_two_launches_and_raise(monkeypatch):
    envs = _variants(BALANCE4, dict(n_agents=4), 257, monkeypatch, "multidiscrete")
    _assert_one_kernel(envs["one kernel"])
    for bad in [(0, 0, -1), (1, 256, 3), (3, 100, -(2 ** 40))]:
        _run(envs, steps=2, reset_at=-1, bad_at=(1, bad))
    envs = _variants(BALANCE3, dict(n_agents=3), 257, monkeypatch, "continuous")
    for bad in [(0, 3, float("nan")), (2, 200, float("nan"))]:
        _run(envs, steps=2, reset_at=-1, bad_at=(1, bad))


def test_batches_on_each_lane_mapping_and_past_the_gpu(monkeypatch):
    """Transport with 2 lines and 3 substeps has a grid barrier: lane pairs while the blocks fit the GPU twice over,
    one lane per env up to what fits once, then the ingest launch in front of the whole-step kernel."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kwargs = dict(n_agents=4, n_lines=2, substeps=3)
    for n, launches in ((sms * 8 * 64 // 2 + 64, 1), (sms * 8 * 64 + 64 * 16, 2)):
        envs = _variants(TRANSPORT, kwargs, n, monkeypatch, "continuous", two_launches=False)
        _assert_one_kernel(envs["one kernel"])
        one = envs["one kernel"]
        backend = one.world._get_backend()
        sync_env(envs["eager"], one)
        gen = torch.Generator().manual_seed(3)
        for t in range(3):
            actions = _actions(one, gen)
            want = envs["eager"].step([a.clone() for a in actions])
            before = backend.launches
            got = one.step([a.clone() for a in actions])
            assert (backend.launches - before == 1) == (launches == 1), f"{n} envs step {t}"
            _check(got, want, one, envs["eager"], f"{n} envs step {t}")
        del envs


def test_sixteen_bit_observations(monkeypatch):
    envs = _variants(BALANCE4, dict(n_agents=4), 1001, monkeypatch, "continuous", obs_dtype=torch.float16)
    _assert_one_kernel(envs["one kernel"])
    _run(envs)


def test_bicycles_stay_on_two_launches(monkeypatch):
    envs = _variants(_with_models(balance.Scenario, balance, ["bicycle", "holo"]), dict(n_agents=2), 129, monkeypatch,
                     "continuous", two_launches=False)
    assert envs["one kernel"]._one_call.c.ingest_in_kernel == 0
    _run(envs, steps=4, reset_at=2)
