"""The action ingest on every CUDA path, at its edges, against the float64 reference (tests/action_ref.py) with the
cases of tests/action_cases.py:

(a) ``ingest_actions_kernel<false>`` (holonomic agents only), (b) ``<true>`` (the same plus a kinematic agent),
(c) ``ingest_broad_kernel`` (eager balance), (d) the prologue of the one-kernel step (balance, 3 and 4 agents,
lane pairs at 1001 envs and one thread per env at a batch between the two capacities), (e) the torch path on CUDA
(``action_checks="sync"``), (f) pinned host actions into (a) and (d).

Decoded actions and holonomic forces are bit-exact; the deferred check raises exactly when the reference asserts
(any NaN, or |clamp(v)| > u_range).  A legal batch holding every edge value goes first: it must not raise.
"""
import math

import numpy as np
import pytest
import torch

import action_cases as cases
import action_ref as ref
import vectorizedmultiagentsimulator_b200 as b200
from test_action_ingest_hostsim import _kin_ref, _within, assert_bits, kinematic_inputs

pytestmark = pytest.mark.gpu


def _ranges(agent):
    return agent.action.u_range_tensor.cpu().numpy(), agent.action.u_multiplier_tensor.cpu().numpy()


def _check_decoded(env, actions, clamp, what):
    for i, (agent, a) in enumerate(zip(env.agents, actions)):
        r, m = _ranges(agent)
        want, _ = ref.continuous(a, r, m, clamp)
        assert_bits(agent.action.u.cpu().numpy(), want, f"{what}: agent {i} u")
        model = type(agent.dynamics).__name__
        if model.startswith("Holonomic"):
            assert_bits(agent.state.force.cpu().numpy(), want[:, :2], f"{what}: agent {i} force")
            if model == "HolonomicWithRotation":
                assert_bits(agent.state.torque.cpu().numpy()[:, 0], want[:, 2], f"{what}: agent {i} torque")


def _raises_iff(env, flagged, what):
    if flagged:
        with pytest.raises(AssertionError):
            env.check_actions_now()
    else:
        env.check_actions_now()
    env.check_actions_now()  # (the flag was cleared by the raise)


def _sweep(env, legal, clamp, run, targets, what):
    """Each bad value alone at (agent, component, env) of ``targets``; ``run(actions)`` ingests them."""
    for i, j, e in targets:
        r, m = _ranges(env.agents[i])
        for v in cases.edge_values(r[j])[1] + cases.edge_values(r[j])[2]:
            acts = [a.copy() for a in legal]
            acts[i][e, j] = v
            run(acts)
            want, flagged = ref.continuous(acts[i], r, m, clamp)
            _raises_iff(env, bool(flagged.any()), f"{what}: agent {i} component {j} env {e} value {v}")
            u = env.agents[i].action.u.cpu().numpy()
            assert_bits(u[e], want[e], f"{what}: agent {i} component {j} env {e} value {v}")


def _legal(env, clamp, seed=3):
    rng = np.random.default_rng(seed)
    return [cases.legal_batch(_ranges(a)[0], clamp, env.num_envs, rng) for a in env.agents]


def _eager(env, pinned=False):
    def run(acts):
        ts = [torch.from_numpy(a) for a in acts]
        ts = [t.pin_memory() for t in ts] if pinned else [t.cuda() for t in ts]
        assert env._fused_ingest_applies(ts)
        env._apply_actions(ts)
        torch.cuda.synchronize()
    return run


def _holo_env(clamp, B=517, kin=None, extra_agents=(), **kw):
    """Agents with 2 (Holonomic), 3 (HolonomicWithRotation) and 8 action components, every range and multiplier."""
    r8, m8 = cases.agent_layouts()[-1]
    agents = [("holo", cases.RANGES[:2], [0.7, 0.01], None), ("holo_rot", cases.RANGES[1:], [0.01, 0.7, 1.0], None),
              ("holo", r8, m8, None)]
    if kin is not None:
        agents.append(kin)
    agents += list(extra_agents)
    return b200.make_env(cases.make_scenario(agents, kw.pop("dt", 0.1)), num_envs=B, device="cuda", seed=0,
                         clamp_actions=clamp, **kw)


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("clamp", [False, True])
def test_eager_ingest_of_holonomic_agents(clamp, pinned):
    """(a), (f): ingest_actions_kernel<false>; the size-8 agent and partial last block (517 envs)."""
    env = _holo_env(clamp)
    B = env.num_envs
    legal = _legal(env, clamp)
    run = _eager(env, pinned)
    run(legal)
    _check_decoded(env, legal, clamp, "legal batch")
    env.check_actions_now()
    _sweep(env, legal, clamp, run, [(0, 0, 0), (1, 2, B - 1), (2, 7, B - 3), (2, 3, 0)], "eager")


@pytest.mark.parametrize("kind", ["diff", "bicycle", "drone"])
@pytest.mark.parametrize("dt", cases.DTS)
def test_kinematic_instantiation_decodes_holonomic_agents_and_models(kind, dt):
    """(b): ingest_actions_kernel<true>: the holonomic agents decode as in (a), the kinematic model is within 4x the
    fp32 bound of float64 (RK4 and Euler)."""
    for rk4 in (True, False):
        u, rot, pos, vel, ang_vel, state = kinematic_inputs(kind, dt, rk4)
        B = u.shape[0]
        size, _, agent_kw, model_kw = cases.KIN[kind]
        kin = (kind, [1e30] * size, [1.0] * size, (agent_kw, model_kw, "rk4" if rk4 else "euler"))
        env = _holo_env(False, B=B, kin=kin, dt=dt)
        agent = env.agents[-1]
        agent.set_pos(torch.from_numpy(pos).cuda(), batch_index=None)
        agent.set_vel(torch.from_numpy(vel).cuda(), batch_index=None)
        agent.set_rot(torch.from_numpy(rot)[:, None].cuda(), batch_index=None)
        agent.set_ang_vel(torch.from_numpy(ang_vel)[:, None].cuda(), batch_index=None)
        if state is not None:
            agent.dynamics.drone_state.copy_(torch.from_numpy(state))
        legal = _legal(env, False)[:-1]
        acts = [torch.from_numpy(a).cuda() for a in legal] + [torch.from_numpy(u).cuda()]
        assert env._fused_ingest_applies(acts)
        env._apply_actions(acts)
        torch.cuda.synchronize()
        env.check_actions_now()
        _check_decoded(env, legal, False, "holonomic agents beside a kinematic one")
        u_out, new_state, fx, fy, t = _kin_ref(kind, u, rot, pos, vel, ang_vel, state, dt, rk4)
        what = f"{kind} dt={dt} rk4={rk4}"
        _within(agent.state.force[:, 0].cpu().numpy(), fx, what + " force x")
        _within(agent.state.force[:, 1].cpu().numpy(), fy, what + " force y")
        _within(agent.state.torque[:, 0].cpu().numpy(), t, what + " torque")
        if kind == "drone":
            _within(agent.action.u.cpu().numpy(), u_out, what + " u")
            _within(agent.dynamics.drone_state.cpu().numpy(), new_state, what + " drone state")


@pytest.mark.parametrize("clamp", [False, True])
def test_ingest_with_the_broad_phase_in_one_launch(clamp):
    """(c): eager balance (masked pairs, no pre_step override): ingest_broad_kernel."""
    env = b200.make_env("balance", num_envs=1001, device="cuda", seed=0, n_agents=4, clamp_actions=clamp)
    env.reset()
    legal = _legal(env, clamp)
    run = _eager(env)
    run(legal)
    assert env.world._get_backend()._mask_ready, "the ingest must have built the broad-phase mask"
    _check_decoded(env, legal, clamp, "balance eager")
    env.check_actions_now()
    _sweep(env, legal, clamp, run, [(0, 0, 0), (3, 1, 1000), (1, 1, 999)], "balance eager")


def _one_kernel_env(n_agents, B, clamp):
    env = b200.make_env("balance", num_envs=B, device="cuda", seed=0, cuda_graph=True, n_agents=n_agents,
                        clamp_actions=clamp)
    env.reset()
    for _ in range(4):
        env.step([torch.zeros(B, 2, device="cuda") for _ in range(n_agents)])
    assert env._one_call_state == "on" and env._one_call.c.ingest_in_kernel == 1 and env._one_call.c.fused_kernel > 0
    return env


@pytest.mark.parametrize("clamp", [False, True])
@pytest.mark.parametrize("n_agents", [3, 4])
@pytest.mark.parametrize("lanes", [2, 1])
def test_one_kernel_step_prologue(lanes, n_agents, clamp):
    """(d), (f): the whole step as one launch.  Lane pairs (G = 2) at 1001 envs: the odd lane's agent and the last,
    partial pair; one thread per env (G = 1) between SMs x 4 x 64 and SMs x 8 x 64 envs."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 1001 if lanes == 2 else sms * 4 * 64 + 1001
    env = _one_kernel_env(n_agents, B, clamp)
    legal = _legal(env, clamp)
    steps = env.steps.clone()
    backend = env.world._get_backend()
    before = backend.launches
    env.step([torch.from_numpy(a).cuda() for a in legal])
    assert backend.launches - before == 1, "the step must be one launch"
    assert torch.equal(env.steps, steps + 1), "the step counter advances once"
    _check_decoded(env, legal, clamp, f"one kernel G={lanes}")
    env.check_actions_now()
    # pinned host actions, read by the prologue where they lie
    env.step([torch.from_numpy(a).pin_memory() for a in legal])
    torch.cuda.synchronize()
    _check_decoded(env, legal, clamp, f"one kernel G={lanes}, pinned")
    env.check_actions_now()

    def run(acts):
        before = backend.launches
        env.step([torch.from_numpy(a).cuda() for a in acts])
        torch.cuda.synchronize()
        assert backend.launches - before == 1

    _sweep(env, legal, clamp, run, [(0, 0, 0), (1, 1, B - 1), (1, 0, B - 2), (n_agents - 1, 1, 64)],
           f"one kernel G={lanes}")


@pytest.mark.parametrize("clamp", [False, True])
def test_torch_path_on_cuda(clamp):
    """(e): action_checks="sync": the torch statements on CUDA assert at once."""
    env = _holo_env(clamp, B=129, action_checks="sync")
    legal = _legal(env, clamp)
    env._apply_actions([torch.from_numpy(a).cuda() for a in legal])
    _check_decoded(env, legal, clamp, "torch on cuda")
    for i, j in ((0, 1), (2, 7)):
        r, m = _ranges(env.agents[i])
        for v in cases.bad_values(r[j], clamp):
            acts = [a.copy() for a in legal]
            acts[i][-1, j] = v
            _, flagged = ref.continuous(acts[i], r, m, clamp)
            assert flagged.any()
            with pytest.raises(AssertionError):
                env._apply_actions([torch.from_numpy(a).cuda() for a in acts])


def test_more_than_16_agents_and_a_9_component_agent():
    """18 agents: the ingest is split into launches and the step counter still advances once per step; an agent with
    9 action components is decoded by the torch path, to the same bits."""
    nine = ("holo", [1.0, 0.7, 1e-4, 3.0, 1.0, 0.7, 1e-4, 3.0, 1.0], [0.7] * 9, None)
    many = [("holo", [1.0, 0.7], [0.7, 0.01], None) for _ in range(18)]
    for agents, fused in ((many, True), ([nine] + many[:2], False)):
        env = b200.make_env(cases.make_scenario(agents), num_envs=257, device="cuda", seed=0, clamp_actions=True)
        legal = _legal(env, True)
        acts = [torch.from_numpy(a).cuda() for a in legal]
        assert env._fused_ingest_applies(acts) == fused
        steps = env.steps.clone()
        env.step(acts)
        torch.cuda.synchronize()
        assert torch.equal(env.steps, steps + 1)
        _check_decoded(env, legal, True, f"{len(agents)} agents")
        env.check_actions_now()
        acts[-1][5, 1] = math.nan
        env.step(acts)
        with pytest.raises(AssertionError):
            env.check_actions_now()
