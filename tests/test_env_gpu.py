"""End-to-end parity on the GPU: ``make_env(...).step`` on CUDA vs the same env on the CPU oracle.

The CPU-oracle env is itself pinned against the unmodified reference in
tests/test_env_vs_reference.py (bit-equal obs / rewards / dones); here the CUDA env is compared
with it teacher-forced (state re-synchronised before every step) and in a short free roll-out.
"""
import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from oracle.backend import use_oracle
from vectorizedmultiagentsimulator_b200 import _native

#: two different kernels running the same arithmetic give the same bits in the exact build; in the opt-in
#: fast-arithmetic build the compiler contracts and approximates per kernel, so there they are compared from
#: a common state every step (``resync``) and to the parity tolerance (``same``)
EXACT = _native.ARITH == "exact"


def same(got, want):
    return same_result(got, want, atol=2e-4)


def resync(reference, *others):
    if not EXACT:
        for other in others:
            sync_env(reference, other)

pytestmark = pytest.mark.gpu

CASES = [
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3)),  # BASELINE.json configs[2] variant
    ("navigation", dict(n_agents=8)),
    ("flocking", dict(n_agents=5)),
]


def _make_pair(name, kwargs, n_envs):
    with use_oracle():
        cpu = b200.make_env(name, num_envs=n_envs, device="cpu", seed=0, **kwargs)
    gpu = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, **kwargs)
    return cpu, gpu


def _compare(got, want, what, atol, rtol=1e-4):
    g, w = flatten(got), flatten(want)
    assert len(g) == len(w), what
    for a, b in zip(g, w):
        a = a.cpu()
        assert a.shape == b.shape and a.dtype == b.dtype, what
        if a.dtype == torch.bool:
            assert torch.equal(a, b), what
        else:
            err = (a - b).abs()
            assert bool((err <= atol + rtol * b.abs()).all()), f"{what}: max |err| {float(err.max())}"


@pytest.mark.parametrize("name,kwargs", CASES)
def test_env_step_teacher_forced(name, kwargs):
    n_envs = 64
    cpu, gpu = _make_pair(name, kwargs, n_envs)
    gen = torch.Generator().manual_seed(7)
    for t in range(12):
        sync_env(cpu, gpu)
        actions = [
            (torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in cpu.agents
        ]
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step([a.to("cuda") for a in actions])
        # rewards are differences of shaping terms ~1e2: compare with an absolute 1e-4
        _compare(got[0], want[0], f"{name} step {t} obs", atol=1e-5)
        _compare(got[1], want[1], f"{name} step {t} rews", atol=2e-4)
        _compare(got[2], want[2], f"{name} step {t} dones", atol=0)
        _compare(got[3], want[3], f"{name} step {t} infos", atol=2e-4)
    gpu.check_actions_now()
    assert gpu.world._get_backend().launches > 0


# BASELINE.json configs[1..4] at their full per-GPU batch sizes
FULL_SIZE_CASES = [
    ("balance", dict(n_agents=4), 32768),
    ("transport", dict(n_agents=4, n_lines=2, substeps=3), 16384),
    ("navigation", dict(n_agents=8), 8192),  # incl. the LIDAR readings in the observations
    ("flocking", dict(n_agents=5), 32768),
]


@pytest.mark.parametrize("name,kwargs,n_envs", FULL_SIZE_CASES)
def test_env_step_teacher_forced_at_baseline_batch_size(name, kwargs, n_envs):
    """The same teacher-forced comparison at the batch sizes BASELINE.json quotes (not a tiled small
    batch: every env has its own reset layout and its own actions), CUDA-graph mode like the bench."""
    with use_oracle():
        cpu = b200.make_env(name, num_envs=n_envs, device="cpu", seed=0, **kwargs)
    gpu = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, cuda_graph=True, **kwargs)
    gen = torch.Generator().manual_seed(13)
    for t in range(4):  # two eager warm-up steps, the capture, one replay
        sync_env(cpu, gpu)
        actions = [
            (torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in cpu.agents
        ]
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step([a.to("cuda") for a in actions])
        _compare(got[0], want[0], f"{name} B={n_envs} step {t} obs", atol=1e-5)
        _compare(got[1], want[1], f"{name} B={n_envs} step {t} rews", atol=2e-4)
        _compare(got[2], want[2], f"{name} B={n_envs} step {t} dones", atol=0)
    gpu.check_actions_now()


@pytest.mark.parametrize("name,kwargs", CASES[:1] + CASES[3:])
def test_env_free_rollout(name, kwargs):
    n_envs = 32
    cpu, gpu = _make_pair(name, kwargs, n_envs)
    sync_env(cpu, gpu)
    gen = torch.Generator().manual_seed(9)
    for t in range(10):
        actions = [
            (torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in cpu.agents
        ]
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step([a.to("cuda") for a in actions])
    _compare(got[0], want[0], f"{name} rollout obs", atol=1e-4)


def test_stock_style_scenario_on_cuda():
    """A scenario in the reference's own style (tests/stock_style.py: per-agent ``is_overlapping`` /
    ``get_distance`` / ``Lidar.measure`` calls, ``torch.cat`` observations, boxes + a line + LIDAR) on
    the CUDA backend against the CPU oracle env, which is bit-equal to the reference for this scenario
    (tests/test_env_vs_reference.py).  Eager mode: boolean-mask indexing (``rew[mask] += c``) syncs with
    the host, so stock code like this cannot be captured in a CUDA graph."""
    import stock_style

    n_envs = 48
    with use_oracle():
        cpu = b200.make_env(stock_style.make_scenario(), num_envs=n_envs, device="cpu", seed=0, n_agents=3)
    gpu = b200.make_env(stock_style.make_scenario(), num_envs=n_envs, device="cuda", seed=0, n_agents=3)
    gen = torch.Generator().manual_seed(5)
    before = gpu.world._get_backend().launches
    for t in range(10):
        sync_env(cpu, gpu)
        actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) for a in cpu.agents]
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step([a.to("cuda") for a in actions])
        _compare(got[0], want[0], f"stock_style step {t} obs", atol=1e-5)
        _compare(got[1], want[1], f"stock_style step {t} rews", atol=1e-4)
        _compare(got[2], want[2], f"stock_style step {t} dones", atol=0)
        _compare(got[3], want[3], f"stock_style step {t} infos", atol=1e-4)
    gpu.check_actions_now()
    assert gpu.world._get_backend().launches > before  # queries, LIDAR and the step ran in libvmas_b200.so


def test_env_scheduling_inside_environment_step(monkeypatch):
    """Periodic env re-ordering (every 2 steps here) in eager and CUDA-graph mode against an env that
    never re-orders: identical observations / rewards / dones."""
    n_envs = 2048
    monkeypatch.setattr(_native, "ENV_REORDER_EVERY", 0)
    plain = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, n_agents=4)
    plain.step(plain.get_random_actions())  # builds its device tables without an order table
    assert plain.world._get_backend()._dev_tables.env_order is None
    monkeypatch.setattr(_native, "ENV_REORDER_EVERY", 2)
    envs = [b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, n_agents=4, cuda_graph=g) for g in (False, True)]
    for env in envs:
        sync_env(plain, env)
    gen = torch.Generator().manual_seed(3)
    for t in range(9):
        actions = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1).cuda() for _ in plain.agents]
        want = plain.step([a.clone() for a in actions])
        for env in envs:
            got = env.step([a.clone() for a in actions])
            for g, w in zip(flatten(got[:3]), flatten(want[:3])):
                assert same(g, w), f"step {t}: re-ordered env differs"
        resync(plain, *envs)
    for env in envs:
        dt = env.world._get_backend()._dev_tables
        assert dt.env_order is not None
        assert torch.equal(torch.sort(dt.env_order.long()).values, torch.arange(n_envs, device="cuda"))


def test_device_side_dynamics_match_the_torch_formulation():
    """SURVEY 8(f)-3: DiffDrive / KinematicBicycle / Drone (RK4 and Euler), Forward, Rotation,
    HolonomicWithRotation and Static run inside the ingest kernel on CUDA.  One agent per model
    (tests/crafted.py "dynamics_zoo"), teacher-forced against the CPU env, whose torch formulation of
    the models is bit-equal to the reference's (tests/test_env_vs_reference.py)."""
    import crafted

    root = "vectorizedmultiagentsimulator_b200"
    n_envs = 96
    with use_oracle():
        cpu = b200.make_env(crafted.make_scenario(root, "dynamics_zoo"), num_envs=n_envs, device="cpu", seed=0)
    gpu = b200.make_env(crafted.make_scenario(root, "dynamics_zoo"), num_envs=n_envs, device="cuda", seed=0)
    assert gpu._fused_ingest_specs() is not None, "the fused ingest kernel must cover every model of the zoo"
    drones = [(a.dynamics, b.dynamics) for a, b in zip(cpu.agents, gpu.agents) if hasattr(a.dynamics, "drone_state")]
    assert drones
    gen = torch.Generator().manual_seed(11)
    launches = gpu.world._get_backend().launches
    for t in range(10):
        sync_env(cpu, gpu)
        for src, dst in drones:
            dst.drone_state = src.drone_state.to("cuda").clone()
        actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in cpu.agents]
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step([a.to("cuda") for a in actions])
        for k in ("force", "torque", "pos", "vel", "rot", "ang_vel"):
            g, w = getattr(gpu.world.slab, k).cpu(), getattr(cpu.world.slab, k)
            err = (g - w).abs()
            assert bool((err <= 1e-5 + 1e-4 * w.abs()).all()), f"step {t} {k}: max |err| {float(err.max())}"
        for src, dst in drones:
            err = (dst.drone_state.cpu() - src.drone_state).abs()
            assert bool((err <= 1e-5 + 1e-4 * src.drone_state.abs()).all()), f"step {t} drone state: {float(err.max())}"
        for a, b in zip(cpu.agents, gpu.agents):  # the scaled actions, incl. the drone's in-place thrust offset
            assert torch.allclose(b.action.u.cpu(), a.action.u, rtol=1e-6, atol=1e-7), f"step {t}: action.u of {a.name}"
        _compare(got[0], want[0], f"dynamics_zoo step {t} obs", atol=1e-5)
    gpu.check_actions_now()
    assert gpu.world._get_backend().launches > launches


@pytest.mark.parametrize("params,form,cutoff", [((2.0, 1.5, 0.02), "standard", 0.3), ((1.2, 0.0, 0.05), "standard", None), ((3.0, 2.0, 0.1), "parallel", None)])
def test_velocity_controller_kernel_equals_the_torch_statements(params, form, cutoff):
    """``VelocityController.process_force`` on CUDA is one kernel (ref controllers/velocity_controller.py:
    113-125); it must reproduce the torch statements it replaces — same fp32 operations, same order."""
    import warnings

    from vectorizedmultiagentsimulator_b200.simulator.controllers.velocity_controller import VelocityController

    env = b200.make_env("navigation", num_envs=257, device="cuda", seed=0, n_agents=2)
    agent = env.world.agents[1]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fused, eager = (VelocityController(agent, env.world, params, form) for _ in range(2))
    eager.use_kernel = False
    for c in (fused, eager):
        if cutoff is not None:
            c.integrator_windup_cutoff = cutoff
    gen = torch.Generator().manual_seed(1)
    before = env.world._get_backend().launches
    for t in range(6):
        agent.set_vel((torch.rand(257, 2, generator=gen) - 0.5).cuda(), batch_index=None)
        target = (torch.rand(257, 2, generator=gen) * 2 - 1).cuda()
        agent.action.u = target.clone()
        fused.process_force()
        got = agent.action.u.clone()
        agent.action.u = target.clone()
        eager.process_force()
        want = agent.action.u
        # torch's CUDA `tensor / python_scalar` multiplies by the reciprocal, the kernel divides (like torch on
        # the CPU): equal to an ulp or two, not bit for bit
        close = lambda a, b: torch.allclose(a, b, rtol=2e-6, atol=1e-6)  # noqa: E731
        assert close(got, want), f"iteration {t}: max |diff| {float((got - want).abs().max())}"
        assert close(fused.accum_errs, eager.accum_errs) and close(fused.prev_err, eager.prev_err)
    assert env.world._get_backend().launches == before + 6


@pytest.mark.parametrize("multidiscrete", [False, True])
@pytest.mark.parametrize("name,kwargs", [("balance", dict(n_agents=3)), ("navigation", dict(n_agents=4))])
def test_discrete_actions_decoded_on_the_device(name, kwargs, multidiscrete):
    """Discrete and multi-discrete action spaces (ref environment.py:656-706) go through the fused ingest
    kernel too: flat index -> per-component index -> force level, incl. the odd-n re-ordering.  Teacher-forced
    against the CPU env (whose torch decoding is bit-equal to the reference's, tests/test_env_vs_reference.py)."""
    n_envs = 128
    opts = dict(continuous_actions=False, multidiscrete_actions=multidiscrete, **kwargs)
    with use_oracle():
        cpu = b200.make_env(name, num_envs=n_envs, device="cpu", seed=0, **opts)
    gpu = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, **opts)
    gen = torch.Generator().manual_seed(21)
    for t in range(6):
        sync_env(cpu, gpu)
        if multidiscrete:
            actions = [torch.stack([torch.randint(0, n, (n_envs,), generator=gen) for n in a.discrete_action_nvec], dim=-1) for a in cpu.agents]
        else:
            actions = [torch.randint(0, 9, (n_envs, 1), generator=gen) for _ in cpu.agents]
        gpu_actions = [a.cuda() for a in actions]
        assert gpu._fused_ingest_applies(gpu_actions), "discrete actions must take the fused ingest kernel"
        want = cpu.step([a.clone() for a in actions])
        got = gpu.step(gpu_actions)
        for a_cpu, a_gpu in zip(cpu.agents, gpu.agents):
            assert torch.equal(a_gpu.action.u.cpu(), a_cpu.action.u), f"step {t}: decoded action of {a_cpu.name}"
        _compare(got[0], want[0], f"{name} discrete step {t} obs", atol=1e-5)
        _compare(got[1], want[1], f"{name} discrete step {t} rews", atol=2e-4)
    gpu.check_actions_now()
    bad = [torch.full((n_envs, a.action_size if multidiscrete else 1), 99, dtype=torch.int64, device="cuda") for a in gpu.agents]
    gpu.step(bad)  # out of range: flagged on the device, raised by the deferred check
    torch.cuda.synchronize()
    with pytest.raises(AssertionError):
        gpu.check_actions_now()


@pytest.mark.parametrize("graph", [False, True])
def test_broad_phase_in_the_ingest_launch_changes_no_bit(graph):
    """The action ingest also builds the coming step's first broad-phase mask (one launch instead of two)
    when nothing can move an entity in between; a scenario that overrides ``pre_step`` keeps the separate
    launch.  Same roll-out either way, bit for bit (balance: line / box pairs obey the mask)."""
    n_envs = 640
    fused = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, n_agents=4, cuda_graph=graph)
    plain = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, n_agents=4, cuda_graph=graph)
    plain.scenario.__class__ = type("WithPreStep", (plain.scenario.__class__,), {"pre_step": lambda self: None})
    sync_env(fused, plain)
    gen = torch.Generator().manual_seed(17)
    counts = []
    for t in range(8):
        actions = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1).cuda() for _ in fused.agents]
        before = [e.world._get_backend().launches for e in (fused, plain)]
        got = fused.step([a.clone() for a in actions])
        want = plain.step([a.clone() for a in actions])
        counts.append([e.world._get_backend().launches - b for e, b in zip((fused, plain), before)])
        for g, w in zip(flatten(got[:3]), flatten(want[:3])):
            assert same(g, w), f"step {t}"
        resync(plain, fused)
    if graph:
        # captured: the whole step is ONE kernel; with pre_step overridden the ingest and the broad phase stay
        # launches of their own in front of the whole-step kernel
        assert counts[-3:] == [[1, 3]] * 3, counts
    else:
        assert all(c[1] == c[0] + 1 for c in counts[-3:]), counts  # the separate broad-phase launch


def test_reset_at_and_state_views_on_gpu():
    env = b200.make_env("transport", num_envs=8, device="cuda", seed=0, n_agents=3)
    agent = env.world.agents[0]
    pos_view = agent.state.pos
    env.step(env.get_random_actions())
    assert pos_view.data_ptr() == agent.state.pos.data_ptr(), "state must stay a view into the slab"
    before = env.world.slab.pos.clone()
    env.reset_at(3)
    after = env.world.slab.pos
    changed = (before != after).flatten(1).any(1)
    assert bool(changed[3]) and not bool(changed[[0, 1, 2, 4, 5, 6, 7]].any())
    # in-place row write through the getter view lands in the slab
    agent.state.pos[2] = torch.tensor([0.25, -0.5], device="cuda")
    assert torch.equal(env.world.slab.pos[2, env.world.entities.index(agent)].cpu(), torch.tensor([0.25, -0.5]))


def test_cpu_world_refuses_to_step():
    env_world_error = None
    try:
        b200.make_env("balance", num_envs=2, device="cpu", seed=0)
    except RuntimeError as err:  # the first observation needs is_overlapping -> CUDA only
        env_world_error = str(err)
    assert env_world_error and "no CPU fallback" in env_world_error


def test_deferred_action_check_raises_next_step():
    env = b200.make_env("navigation", num_envs=4, device="cuda", seed=0, n_agents=2)
    bad = [torch.full((4, 2), 5.0, device="cuda") for _ in env.agents]
    env.step(bad)  # flagged on the device, raised by a later call once the read-back has landed
    torch.cuda.synchronize()
    with pytest.raises(AssertionError):
        env.step(env.get_random_actions())
    env.step(bad)
    with pytest.raises(AssertionError):
        env.check_actions_now()  # deterministic variant: waits for the flag


@pytest.mark.parametrize("name,kwargs", CASES)
def test_cuda_graph_mode_is_bit_identical_to_eager(name, kwargs):
    """cuda_graph=True replays the captured step; results must equal the eager path bit for bit,
    across partial and full resets executed between replays."""
    n_envs = 48
    eager = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, **kwargs)
    graph = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, cuda_graph=True, **kwargs)
    sync_env(eager, graph)
    gen = torch.Generator().manual_seed(3)
    for t in range(9):
        actions = [
            ((torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor.cpu()).cuda()
            for a in eager.agents
        ]
        want = eager.step([a.clone() for a in actions])
        got = graph.step([a.clone() for a in actions])
        for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
            assert g.is_contiguous(), f"{name}: output {i} is not contiguous"
            diff = float((g.float() - w.float()).abs().max())
            assert same(g, w), f"{name} step {t} output {i} shape {tuple(g.shape)} max diff {diff}"
        resync(eager, graph)
        if t == 4:
            eager.reset_at(5)
            graph.reset_at(5)
            sync_env(eager, graph)
        if t == 6:
            eager.reset()
            graph.reset()
            sync_env(eager, graph)
    assert graph.graph_replays >= 6
    # every shipped scenario's captured step goes through the one-call entry point (vmas_b200_env_step)
    assert graph._one_call_state == "on", f"{name}: captured step not on vmas_b200_env_step"
    # outputs of one step must survive the next replay (they are clones of the static buffers)
    kept = [o.clone() for o in got[0]]
    graph.step([a.clone() for a in actions])
    for a, b in zip(kept, got[0]):
        assert torch.equal(a, b)


def test_graph_mode_outputs_are_freed_by_refcount():
    """Dropped step outputs must return to the allocator at once (no reference cycle that waits
    for the cyclic GC): otherwise every step of a training loop allocates fresh device memory."""
    import gc

    env = b200.make_env("balance", num_envs=4096, device="cuda", seed=0, cuda_graph=True, n_agents=4)
    env.reset()
    actions = env.get_random_actions()
    for _ in range(5):
        env.step(actions)
    gc.collect()
    gc.disable()
    try:
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        for _ in range(20):
            env.step(actions)
        torch.cuda.synchronize()
        after = torch.cuda.memory_allocated()
    finally:
        gc.enable()
    assert after <= before + (1 << 16), f"graph-mode steps leak device memory: {before} -> {after} bytes"


def test_a_graph_that_draws_device_random_numbers_stays_on_torchs_replay():
    """vmas_b200_env_step launches the captured graph itself; torch's replay additionally advances the
    philox offset of a graph that consumes device random numbers.  Such a graph must not be launched raw
    (it would replay the same numbers): the first replay detects it."""
    from vectorizedmultiagentsimulator_b200.scenarios.balance import Scenario as Balance

    class NoisyBalance(Balance):
        def observation(self, agent):
            obs = super().observation(agent)
            return obs + 0.01 * torch.randn_like(obs)

    env = b200.make_env(NoisyBalance(), num_envs=64, device="cuda", seed=0, cuda_graph=True, n_agents=3)
    env.reset()
    seen = []
    for _ in range(6):
        obs = env.step(env.get_random_actions())[0]
        seen.append(obs[0].clone())
    assert env.graph_replays >= 3
    assert env._one_call_state == "off"
    noise = [(a - b).abs().max().item() for a, b in zip(seen[-2:], seen[-3:-1])]
    assert all(n > 0 for n in noise)

    quiet = b200.make_env("balance", num_envs=64, device="cuda", seed=0, cuda_graph=True, n_agents=3)
    quiet.reset()
    for _ in range(6):
        quiet.step(quiet.get_random_actions())
    assert quiet._one_call_state == "on"


def test_every_way_of_issuing_a_captured_step_gives_the_same_bits(monkeypatch):
    """balance's captured step holds only library launches, so it runs as ONE kernel (action ingest + broad
    phase with a grid-wide barrier + substeps + step program + observation rows, results written straight
    into the step's fresh output tensors; vmas_b200_env_step, direct mode).  The same step with the ingest as
    a launch of its own,  The same step with the results copied out of
    static buffers, as two launches (no whole-step kernel), as a graph launch from the library, as torch's
    replay with separate ingest / hand-out calls, and eagerly must all give the same bits."""
    from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

    variants = {
        "one kernel": dict(),
        "whole-step kernel": dict(_INGEST_IN_KERNEL=False),
        "copied results": dict(_WRITE_RESULTS_IN_PLACE=False),
        "two launches": dict(_WHOLE_STEP_KERNEL=False),
        "graph launch": dict(_DIRECT_STEP=False),
        "torch replay": dict(_ONE_CALL_STEP=False),
    }
    envs = {}
    for label, flags in variants.items():
        with monkeypatch.context() as m:
            for k, v in flags.items():
                m.setattr(E, k, v)
            env = b200.make_env("balance", num_envs=96, device="cuda", seed=0, cuda_graph=True, n_agents=4)
            env.reset()
            # (the flags are read when the step is captured: warm-up steps + capture happen here)
            for _ in range(4):
                env.step([torch.zeros(96, 2, device="cuda") for _ in range(4)])
            envs[label] = env
    eager = b200.make_env("balance", num_envs=96, device="cuda", seed=0, n_agents=4)
    eager.reset()
    for _ in range(4):
        eager.step([torch.zeros(96, 2, device="cuda") for _ in range(4)])
    for env in envs.values():
        sync_env(eager, env)
    gen = torch.Generator().manual_seed(5)
    for t in range(10):
        actions = [(torch.rand(96, 2, generator=gen) * 2 - 1).cuda() for _ in range(4)]
        want = eager.step([x.clone() for x in actions])
        for label, env in envs.items():
            got = env.step([x.clone() for x in actions])
            for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
                assert same(g, w), f"{label}: step {t} output {i}"
            for k in ("pos", "vel", "rot", "ang_vel"):
                assert same(getattr(env.world.slab, k), getattr(eager.world.slab, k)), f"{label}: step {t} {k}"
        resync(eager, *envs.values())
        if t == 5:  # a partial reset in between (the carried shaping term is rewritten in place)
            eager.reset_at(7)
            for env in envs.values():
                env.reset_at(7)
                sync_env(eager, env)
    one, whole, copied, two, graph, replay = (envs[k] for k in variants)
    assert one._one_call.c.ingest_in_kernel == 1 and one._one_call.c.fused_kernel > 0 and one._one_call.c.n_segs == 0
    assert whole._one_call.c.ingest_in_kernel == 0
    assert whole._one_call_state == "on" and whole._one_call.direct and whole._one_call.c.fused_kernel > 0
    assert whole._one_call.c.n_segs == 0 and whole._one_call.c.obs_block >= 0 and whole._one_call.c.n_mirrors == 13
    assert copied._one_call.c.fused_kernel > 0 and copied._one_call.c.n_segs >= 14 and copied._one_call.c.n_mirrors == 0
    assert two._one_call_state == "on" and two._one_call.direct and two._one_call.c.fused_kernel == 0
    assert graph._one_call_state == "on" and not graph._one_call.direct
    assert replay._one_call_state == "off"
    assert float(whole.steps[0]) == float(eager.steps[0])
    # kernels per step: ingest (+ broad phase) and the whole-step kernel; with copied results the hand-out copy
    for env, n in ((one, 1), (whole, 2), (copied, 2), (two, 3)):
        before = env.world._get_backend().launches
        env.step(actions)
        assert env.world._get_backend().launches - before == n


def test_one_kernel_step_falls_back_when_the_batch_does_not_fit_the_gpu_at_once():
    """The one-kernel step's broad phase needs a grid-wide barrier, hence every block resident; beyond that
    (here: more envs than the GPU's SMs x 8 blocks x 64 threads) the same call issues ingest + whole-step kernel."""
    n_envs = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 64 + 4096
    big = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, cuda_graph=True, n_agents=4)
    eager = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, n_agents=4)
    big.reset()
    eager.reset()
    sync_env(eager, big)
    gen = torch.Generator().manual_seed(11)
    for t in range(7):
        actions = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1).cuda() for _ in range(4)]
        want = eager.step([x.clone() for x in actions])
        got = big.step([x.clone() for x in actions])
        for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
            assert same(g, w), f"step {t} output {i}"
        resync(eager, big)
    assert big._one_call_state == "on" and big._one_call.c.ingest_in_kernel == 1
    before = big.world._get_backend().launches
    big.step(actions)
    assert big.world._get_backend().launches - before == 2


@pytest.mark.parametrize("graph", [False, True])
def test_pinned_host_actions_are_read_where_they_lie(graph):
    """Continuous actions handed in as PINNED host tensors are not staged: the ingest (a launch of its own, or
    the prologue of the one-kernel step) reads them over PCIe.  Same results as with device tensors."""
    n_envs = 256
    a = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, cuda_graph=graph, n_agents=4)
    b = b200.make_env("balance", num_envs=n_envs, device="cuda", seed=0, cuda_graph=graph, n_agents=4)
    sync_env(a, b)
    gen = torch.Generator().manual_seed(23)
    for t in range(7):
        host = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1).pin_memory() for _ in range(4)]
        assert a._fused_ingest_applies(host)
        got = a.step(host)
        want = b.step([x.cuda() for x in host])
        torch.cuda.synchronize()
        for g, w in zip(flatten(got), flatten(want)):
            assert torch.equal(g, w), f"step {t}"
        for ag_a, ag_b in zip(a.agents, b.agents):
            assert torch.equal(ag_a.action.u, ag_b.action.u)
    if graph:
        assert a._one_call_state == "on"


@pytest.mark.parametrize(
    "kwargs,launches",
    [
        (dict(n_agents=4), 1),  # the whole step is one kernel
        (dict(n_agents=4, n_lines=2, substeps=3), 1),  # ... with a grid-wide barrier per substep (batch-wide mask)
    ],
)
def test_transport_goal_flags_are_program_results_and_observation_columns(kwargs, launches):
    """transport's ``on_goal`` flags are computed by the step program AND are columns of every agent's
    observation (``observe.value``).  Eagerly that is a program launch followed by a gather launch; captured,
    the whole-step kernel's epilogue reads the flag from the program's register."""
    n_envs = 192
    eager = b200.make_env("transport", num_envs=n_envs, device="cuda", seed=0, **kwargs)
    graph = b200.make_env("transport", num_envs=n_envs, device="cuda", seed=0, cuda_graph=True, **kwargs)
    with use_oracle():
        cpu = b200.make_env("transport", num_envs=n_envs, device="cpu", seed=0, **kwargs)
    # put a package on its goal in a few envs so that the flag is not constant
    for env in (cpu, eager, graph):
        package, goal = env.scenario.packages[0], env.world.landmarks[0]
        sync_env(cpu, env) if env is not cpu else None
    pos = cpu.scenario.packages[0].state.pos.clone()
    pos[::5] = cpu.world.landmarks[0].state.pos[::5]
    for env in (cpu, eager, graph):
        env.scenario.packages[0].set_pos(pos.to(env.device), batch_index=None)
    gen = torch.Generator().manual_seed(9)
    for t in range(8):
        actions = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1) for _ in cpu.agents]
        want = eager.step([a.cuda() for a in actions])
        got = graph.step([a.cuda() for a in actions])
        ref = cpu.step([a.clone() for a in actions])
        for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
            assert same(g, w), f"step {t} output {i}"
        _compare(want[0], ref[0], f"transport step {t} obs vs oracle", atol=1e-5)
        _compare(want[2], ref[2], f"transport step {t} dones vs oracle", atol=0)
        resync(eager, graph)
        sync_env(cpu, eager)
        sync_env(cpu, graph)
    flag_column = want[0][0][:, 4 + 6]  # pos, vel, then per package: 2 + 2 + 2 columns and the flag
    assert 0 < float(flag_column.sum()) < n_envs and set(flag_column.unique().tolist()) <= {0.0, 1.0}
    plan = graph._one_call
    assert graph._one_call_state == "on" and plan.direct and plan.c.fused_kernel > 0
    before = graph.world._get_backend().launches
    graph.step([a.cuda() for a in actions])
    assert graph.world._get_backend().launches - before == launches


def test_value_columns_without_a_whole_step_kernel_keep_the_captured_graph(monkeypatch):
    """Observation columns fed by the step program need program and gather in one thread (the whole-step
    kernel) or in two launches; without the kernel (no compiler on the box, or switched off) the captured
    step must stay a graph holding the two launches — never the single fused launch, which would race."""
    from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

    monkeypatch.setattr(E, "_WHOLE_STEP_KERNEL", False)
    n_envs = 128
    eager = b200.make_env("transport", num_envs=n_envs, device="cuda", seed=0, n_agents=3)
    graph = b200.make_env("transport", num_envs=n_envs, device="cuda", seed=0, n_agents=3, cuda_graph=True)
    sync_env(eager, graph)
    gen = torch.Generator().manual_seed(2)
    for t in range(7):
        actions = [(torch.rand(n_envs, 2, generator=gen) * 2 - 1).cuda() for _ in eager.agents]
        want = eager.step([a.clone() for a in actions])
        got = graph.step([a.clone() for a in actions])
        for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
            assert same(g, w), f"step {t} output {i}"
        resync(eager, graph)
    assert graph._one_call_state == "on" and not graph._one_call.direct and graph._one_call.c.fused_kernel == 0
