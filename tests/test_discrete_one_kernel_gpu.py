"""The captured step of a discrete or multi-discrete action space as ONE launch (``step_env_kernel`` with the
discrete action prologue): it must return, bit for bit, what the eager step and the two-launch captured step
(ingest kernel, then the whole-step kernel; ``_INGEST_IN_KERNEL = False``) return — observations, rewards, dones,
infos, the physics state and ``agent.action.u`` — and flag the same illegal indices.

Covered: balance with 3 and 4 agents (a lone agent on a lane pair), transport with 4 agents and with 2 lines and 3
substeps (the batch-wide broad phase behind a grid barrier), a scenario with non-default ``discrete_action_nvec``,
asymmetric ``u_range`` and ``u_multiplier != 1``, batches on each lane mapping (G = 2, G = 1) and one past what the
GPU holds at once (two launches again, same bits), and 16-bit observations.
"""
import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.scenarios import balance
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
SLAB = ("pos", "vel", "rot", "ang_vel", "force", "torque")


class SkewedBalance(balance.Scenario):
    """balance whose agents have 5 x 4 choices, asymmetric ranges and multipliers other than 1."""

    def make_world(self, batch_dim, device, **kwargs):
        world = super().make_world(batch_dim, device, **kwargs)
        for i, agent in enumerate(world.agents):
            agent.discrete_action_nvec = [5, 4]
            agent.action._u_range = [0.8, 1.3 + 0.1 * i]
            agent.action._u_multiplier = [0.6, 1.7]
            agent.action._cache.clear()
        return world


def _indices(env, gen, bad=None):
    """Random legal indices per agent ([B, 1] flat or [B, 2] per component), int64 on the device; ``bad``:
    (agent, env, value) written over one of them."""
    out = []
    for agent in env.agents:
        nvec = agent.discrete_action_nvec
        if env.multidiscrete_actions:
            a = torch.stack([torch.randint(0, n, (env.num_envs,), generator=gen) for n in nvec], -1)
        else:
            a = torch.randint(0, nvec[0] * nvec[1], (env.num_envs, 1), generator=gen)
        out.append(a)
    if bad is not None:
        i, e, v = bad
        out[i][e, -1] = v
    return [a.cuda() for a in out]


def _make(scenario, kwargs, n, monkeypatch, multi, flags=None, cuda_graph=True, **env_kw):
    with monkeypatch.context() as m:
        for k, v in (flags or {}).items():
            m.setattr(E, k, v)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)  # (discrete prologues compile when the step is captured)
        if isinstance(scenario, type):  # (a scenario object belongs to one env)
            scenario = scenario()
        env = b200.make_env(scenario, num_envs=n, device="cuda", seed=0, continuous_actions=False,
                            multidiscrete_actions=multi, cuda_graph=cuda_graph, **env_kw, **kwargs)
        env.reset()
        if cuda_graph:  # (the flags are read when the step is captured: warm-up steps + capture happen here)
            gen = torch.Generator().manual_seed(1)
            for _ in range(4):
                env.step(_indices(env, gen))
    return env


def _same(g, w):
    return torch.equal(g, w) if EXACT else same_result(g.float(), w.float(), atol=2e-4)


def _check(got, want, env, ref, what):
    for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
        assert g.dtype == w.dtype and _same(g, w), f"{what}: output leaf {i}"
    for k in SLAB:
        assert _same(getattr(env.world.slab, k), getattr(ref.world.slab, k)), f"{what}: slab {k}"
    for a, b in zip(env.agents, ref.agents):
        assert _same(a.action.u, b.action.u), f"{what}: {a.name} action.u"


def _run(envs, steps=10, n=None, reset_at=5, bad_at=None):
    """Steps every env with the same indices; the first is the reference.  ``bad_at``: (step, (agent, env, value))."""
    ref, *others = envs.values()
    for env in others:
        sync_env(ref, env)
    gen = torch.Generator().manual_seed(7)
    one = envs.get("one kernel")
    for t in range(steps):
        bad = bad_at[1] if bad_at is not None and bad_at[0] == t else None
        actions = _indices(ref, gen, bad)
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


def _variants(scenario, kwargs, n, monkeypatch, multi, two_launches=True, **env_kw):
    envs = {
        "eager": _make(scenario, kwargs, n, monkeypatch, multi, cuda_graph=False, **env_kw),
        "one kernel": _make(scenario, kwargs, n, monkeypatch, multi, **env_kw),
    }
    if two_launches:
        envs["two launches"] = _make(scenario, kwargs, n, monkeypatch, multi, dict(_INGEST_IN_KERNEL=False), **env_kw)
    return envs


def _assert_one_kernel(env):
    plan = env._one_call
    assert plan is not None and plan.c.ingest_in_kernel == 1 and plan.c.fused_kernel > 0


CASES = [
    ("balance", dict(n_agents=3)),
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3)),
]


@pytest.mark.parametrize("multi", [False, True], ids=["discrete", "multidiscrete"])
@pytest.mark.parametrize("scenario,kwargs", CASES, ids=[f"{s}-{'-'.join(f'{k}{v}' for k, v in kw.items())}" for s, kw in CASES])
def test_one_kernel_step_equals_eager_and_two_launches(scenario, kwargs, multi, monkeypatch):
    envs = _variants(scenario, kwargs, 1001, monkeypatch, multi)  # 1001 envs: lane pairs (G = 2)
    _assert_one_kernel(envs["one kernel"])
    assert envs["two launches"]._one_call.c.ingest_in_kernel == 0
    _run(envs)


@pytest.mark.parametrize("multi", [False, True], ids=["discrete", "multidiscrete"])
def test_non_default_nvec_ranges_and_multipliers(multi, monkeypatch):
    envs = _variants(SkewedBalance, dict(n_agents=3), 333, monkeypatch, multi)
    _assert_one_kernel(envs["one kernel"])
    assert envs["one kernel"].agents[0].discrete_action_nvec == [5, 4]
    _run(envs)


@pytest.mark.parametrize("multi", [False, True], ids=["discrete", "multidiscrete"])
def test_illegal_indices_decode_like_two_launches_and_raise(multi, monkeypatch):
    envs = _variants("balance", dict(n_agents=4), 257, monkeypatch, multi)
    _assert_one_kernel(envs["one kernel"])
    for bad in [(0, 0, -1), (1, 256, 3 if multi else 9), (3, 100, -(2 ** 40)), (2, 5, 2 ** 40)]:
        _run(envs, steps=2, reset_at=-1, bad_at=(1, bad))


def test_batches_on_each_lane_mapping_and_past_the_gpu(monkeypatch):
    """Transport with 2 lines and 3 substeps has a grid barrier: lane pairs while the blocks fit the GPU twice over,
    one lane per env up to what fits once, then the ingest launch in front of the whole-step kernel."""
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    kwargs = dict(n_agents=4, n_lines=2, substeps=3)
    for n, launches in ((sms * 8 * 64 // 2 + 64, 1), (sms * 8 * 64 + 64 * 16, 2)):
        envs = _variants("transport", kwargs, n, monkeypatch, False, two_launches=False)
        _assert_one_kernel(envs["one kernel"])
        one = envs["one kernel"]
        backend = one.world._get_backend()
        sync_env(envs["eager"], one)
        gen = torch.Generator().manual_seed(3)
        for t in range(3):
            actions = _indices(one, gen)
            want = envs["eager"].step([a.clone() for a in actions])
            before = backend.launches
            got = one.step([a.clone() for a in actions])
            assert (backend.launches - before == 1) == (launches == 1), f"{n} envs step {t}"
            _check(got, want, one, envs["eager"], f"{n} envs step {t}")
        del envs


def test_sixteen_bit_observations(monkeypatch):
    envs = _variants("balance", dict(n_agents=4), 1001, monkeypatch, True, obs_dtype=torch.float16)
    _assert_one_kernel(envs["one kernel"])
    _run(envs)
