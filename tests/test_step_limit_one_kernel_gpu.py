"""The captured step of a bounded episode (``max_steps`` and / or ``terminated_truncated=True``) as ONE launch: the
step limit is a step program spliced into the scenario's, and ``step_env_kernel`` takes its count from the prologue.
It must return, bit for bit, what the eager step, the two-launch step (ingest kernel, then the whole-step kernel;
``_INGEST_IN_KERNEL = False``) and the graph replay (``_DIRECT_STEP = False``) return — observations, rewards, dones
or terminated / truncated, infos, ``steps`` and the physics state — and the dones must be the torch statements of
``Environment._done`` over an env without a limit.

Covered: balance with 3 and 4 agents, transport with 4 agents and with 2 lines and 3 substeps; continuous and discrete
actions; ``max_steps`` 1, 5 and 7 with ``terminated_truncated`` off and on, and ``terminated_truncated=True`` without a
limit; staggered counters (envs truncate at different steps); a TorchRL-style loop with ``reset_at(dones)`` between
steps; batches on each lane mapping and past what the GPU holds at once; fp16 observations; two limits in one process.
"""
import gc

import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
SLAB = ("pos", "vel", "rot", "ang_vel", "force", "torque")


def _actions(env, gen):
    out = []
    for agent in env.agents:
        if env.continuous_actions:
            r = agent.action.u_range_tensor.cpu()
            a = (torch.rand(env.num_envs, agent.action_size, generator=gen) * 2 - 1) * r
        else:
            nvec = agent.discrete_action_nvec
            a = torch.randint(0, nvec[0] * nvec[1], (env.num_envs, 1), generator=gen)
        out.append(a.cuda())
    return out


def _make(scenario, kwargs, n, monkeypatch, space, limit, flags=None, cuda_graph=True, **env_kw):
    max_steps, split = limit
    with monkeypatch.context() as m:
        for k, v in (flags or {}).items():
            m.setattr(E, k, v)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)  # (the limit is part of the kernel: compiled at capture)
        env = b200.make_env(scenario, num_envs=n, device="cuda", seed=0, continuous_actions=space == "continuous",
                            cuda_graph=cuda_graph, max_steps=max_steps, terminated_truncated=split, **env_kw, **kwargs)
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
        assert g.dtype == w.dtype and _same(g, w), f"{what}: output leaf {i}"
    assert torch.equal(env.steps, ref.steps), f"{what}: steps"
    for k in SLAB:
        assert _same(getattr(env.world.slab, k), getattr(ref.world.slab, k)), f"{what}: slab {k}"


def _variants(scenario, kwargs, n, monkeypatch, space, limit, two_launches=True, graph=True, **env_kw):
    # the envs of earlier tests go here, not in the middle of a capture below: their teardown makes CUDA calls that a
    # stream capture in torch's global mode refuses
    gc.collect()
    torch.cuda.synchronize()
    envs = {
        "eager": _make(scenario, kwargs, n, monkeypatch, space, limit, cuda_graph=False, **env_kw),
        "one kernel": _make(scenario, kwargs, n, monkeypatch, space, limit, **env_kw),
        # the torch statements' input: an env without a limit hands out the scenario's own dones
        "no limit": _make(scenario, kwargs, n, monkeypatch, space, (None, False), cuda_graph=False, **env_kw),
    }
    if two_launches:
        envs["two launches"] = _make(scenario, kwargs, n, monkeypatch, space, limit, dict(_INGEST_IN_KERNEL=False), **env_kw)
    if graph:
        envs["graph"] = _make(scenario, kwargs, n, monkeypatch, space, limit, dict(_DIRECT_STEP=False), **env_kw)
    return envs


def _assert_one_kernel(env):
    plan = env._one_call
    assert plan is not None and plan.direct and plan.c.ingest_in_kernel == 1 and plan.c.fused_kernel > 0


def _stagger(envs, period):
    ref = envs["eager"]
    ref.steps.copy_((torch.arange(ref.num_envs, dtype=torch.float32) % period).cuda())
    for env in envs.values():
        if env is not ref:
            sync_env(ref, env)


def _dones(ref, out):
    """(terminated, truncated) of a step's results (truncated None without the split)."""
    return (out[2], out[3]) if ref.terminated_truncated else (out[2], None)


def _torch_statements(ref, want, plain):
    """The step's dones against ``Environment._done``'s torch statements over the scenario's own dones ``plain``."""
    terminated, truncated = _dones(ref, want)
    limit = ref.steps >= ref.max_steps if ref.max_steps is not None else None
    if ref.terminated_truncated:
        assert torch.equal(terminated, plain)
        assert torch.equal(truncated, torch.zeros_like(plain) if limit is None else limit)
    else:
        assert torch.equal(terminated, plain + limit)


def _run(envs, steps=9, reset_dones=False):
    """Steps every env with the same actions; "eager" is the reference.  ``reset_dones``: ``reset_at(dones)`` after
    every step (a TorchRL-style loop)."""
    ref, plain = envs["eager"], envs["no limit"]
    gen = torch.Generator().manual_seed(7)
    one = envs["one kernel"]
    finished = 0
    for t in range(steps):
        actions = _actions(ref, gen)
        want = ref.step([a.clone() for a in actions])
        _torch_statements(ref, want, plain.step([a.clone() for a in actions])[2])
        for label, env in envs.items():
            if env is ref or env is plain:
                continue
            backend = env.world._get_backend()
            before = backend.launches
            got = env.step([a.clone() for a in actions])
            if env is one:
                assert backend.launches - before == 1, f"{label} step {t}: {backend.launches - before} launches"
            _check(got, want, env, ref, f"{label} step {t}")
            if not EXACT:
                sync_env(ref, env)
        if not EXACT:
            sync_env(ref, plain)
        if reset_dones:
            terminated, truncated = _dones(ref, want)
            mask = terminated if truncated is None else terminated | truncated
            finished += int(mask.sum())
            want_obs = ref.reset_at(mask)
            assert not bool(ref.steps[mask].any()), f"step {t}: counters of reset envs"
            for label, env in envs.items():
                if env is ref:
                    continue
                got_obs = env.reset_at(mask)
                if env is not plain:
                    for i, (g, w) in enumerate(zip(flatten(got_obs), flatten(want_obs))):
                        assert _same(g, w), f"{label} reset_at obs {i}"
                sync_env(ref, env)
    return finished


MAIN = [
    ("balance", dict(n_agents=3), "continuous", (5, False)),
    ("balance", dict(n_agents=3), "discrete", (7, True)),
    ("balance", dict(n_agents=4), "continuous", (1, True)),
    ("balance", dict(n_agents=4), "discrete", (None, True)),
    ("transport", dict(n_agents=4), "continuous", (7, False)),
    ("transport", dict(n_agents=4), "discrete", (5, True)),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3), "continuous", (5, False)),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3), "discrete", (1, False)),
]


def _id(case):
    scenario, kwargs, space, (max_steps, split) = case
    return f"{scenario}-{'-'.join(f'{k}{v}' for k, v in kwargs.items())}-{space}-max{max_steps}-{'split' if split else 'dones'}"


@pytest.mark.parametrize("scenario,kwargs,space,limit", MAIN, ids=[_id(c) for c in MAIN])
def test_one_kernel_step_equals_eager_two_launches_and_graph(scenario, kwargs, space, limit, monkeypatch):
    envs = _variants(scenario, kwargs, 1001, monkeypatch, space, limit)  # 1001 envs: lane pairs (G = 2)
    _assert_one_kernel(envs["one kernel"])
    assert envs["two launches"]._one_call.c.ingest_in_kernel == 0
    assert envs["graph"]._one_call is None or not envs["graph"]._one_call.direct
    _stagger(envs, 9)
    _run(envs)


@pytest.mark.parametrize("case", [MAIN[0], MAIN[5]], ids=[_id(MAIN[0]), _id(MAIN[5])])
def test_reset_at_dones_between_steps_keeps_one_launch(case, monkeypatch):
    scenario, kwargs, space, limit = case
    envs = _variants(scenario, kwargs, 1001, monkeypatch, space, limit, two_launches=False, graph=False)
    _assert_one_kernel(envs["one kernel"])
    _stagger(envs, limit[0])
    assert _run(envs, steps=12, reset_dones=True) >= 1001  # (every env's episode has ended at least once)
    _assert_one_kernel(envs["one kernel"])


def test_batches_on_each_lane_mapping_and_past_the_gpu(monkeypatch):
    """Transport with 2 lines and 3 substeps has a grid barrier: lane pairs while the blocks fit the GPU twice over,
    one lane per env up to what fits once, then the ingest launch in front of the whole-step kernel."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    scenario, kwargs, space, limit = MAIN[6]
    for n, launches in ((sms * 8 * 64 // 2 + 64, 1), (sms * 8 * 64 + 64 * 16, 2)):
        envs = _variants(scenario, kwargs, n, monkeypatch, space, limit, two_launches=False, graph=False)
        _assert_one_kernel(envs["one kernel"])
        one, ref = envs["one kernel"], envs["eager"]
        _stagger(envs, 6)
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


def test_sixteen_bit_observations(monkeypatch):
    scenario, kwargs, space, limit = MAIN[2]
    envs = _variants(scenario, kwargs, 1001, monkeypatch, space, limit, obs_dtype=torch.float16)
    _assert_one_kernel(envs["one kernel"])
    _stagger(envs, 3)
    _run(envs)


def test_two_limits_in_one_process(monkeypatch):
    scenario, kwargs, space, _ = MAIN[0]
    five = _variants(scenario, kwargs, 1001, monkeypatch, space, (5, False), two_launches=False, graph=False)
    seven = _variants(scenario, kwargs, 1001, monkeypatch, space, (7, False), two_launches=False, graph=False)
    assert five["one kernel"]._one_call.c.fused_kernel != seven["one kernel"]._one_call.c.fused_kernel
    for envs in (five, seven):
        _assert_one_kernel(envs["one kernel"])
        _stagger(envs, 8)
    _run(five, steps=4)
    _run(seven, steps=4)
    _run(five, steps=4)
