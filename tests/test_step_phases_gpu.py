"""The per-entity phases of a substep on every CUDA step kernel, at their edges (the cases of tests/step_cases.py),
against the fp32 oracle and the float64 reference of tests/step_ref.py.

Generic kernels (``mapping=`` ``thread_per_env``, ``lanes_per_env``, ``block_per_env``) through
``_native.world_step`` / ``world_substeps``, the run-time specialised kernel (and its tile kernel where the world
has one: these worlds, without work items, have none), and the
per-env-parameter world through ``vmas_b200_world_step_params``: equal to the oracle (NaN where it has NaN, the same
bits elsewhere, signed zeros included) and within the float64 bound, for whole steps and for substep ranges that
start after substep 0.  Under ``VMAS_B200_ARITH=fast`` only the bound is checked, with division and square root
widened to CUDA's approximate-op error.

End to end: a NaN action with ``clamp_actions=False`` to an agent with ``f_range`` leaves NaN in the force row and in
the agent's velocity, as the CPU oracle env does, and ``check_actions_now()`` raises.
"""
import math

import numpy as np
import pytest
import torch

import step_cases as cases
import step_ref as ref
import vectorizedmultiagentsimulator_b200 as b200
from oracle.backend import use_oracle
from test_step_phases_hostsim import CASES, KEYS, check
from vectorizedmultiagentsimulator_b200 import _native, jit

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
DEVICE = torch.device("cuda:0")


class _Slab:
    def __init__(self, state):
        self.t = {k: torch.from_numpy(np.ascontiguousarray(state[k])).to(DEVICE) for k in KEYS}

    def tensors(self):
        return tuple(self.t[k] for k in KEYS)


def _tables(case, mapping):
    dt = _native.DeviceTables(case.tables, None, DEVICE, mapping=mapping)
    assert dt.mapping == mapping
    params, grav = case.ent_arrays()
    if dt.ent_params is not None:
        dt.ent_params.copy_(torch.from_numpy(params))
    if dt.ent_gravity is not None:
        dt.ent_gravity.copy_(torch.from_numpy(grav))
    return dt


def _run(case, dt, first, n):
    lib = _native.load()
    slab = _Slab(case.state)
    if (first, n) == (0, case.desc.substeps):
        _native.world_step(lib, dt, slab)
    else:
        _native.world_substeps(lib, dt, slab, first, n)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in slab.t.items()}


def _check(got, case, first, n, what):
    if EXACT:
        check(got, case, first, n, what)
        return
    r = case.ref(first, n)
    for k in KEYS:
        g = got[k].astype(np.float64)
        ok = ~r[k].odd
        assert np.isnan(g)[np.isnan(r[k].v)].all(), f"{what} {k}: a NaN was replaced by a number"
        assert (np.abs(g[ok] - r[k].v[ok]) <= r[k].e[ok]).all(), f"{what} {k}: outside the float64 bound"


@pytest.fixture(autouse=True)
def _approx_ops():
    """The fast build divides and takes square roots with CUDA's approximate instructions."""
    old = ref.APPROX
    ref.APPROX = not EXACT
    yield
    ref.APPROX = old


def _specialise(desc):
    if not jit.available():
        pytest.skip("no nvcc / JIT switched off")
    job = jit.request(desc)
    assert job is not None, "the world must be specialisable"
    assert job.done.wait(timeout=600) and job.error is None, job.error
    return job


@pytest.mark.parametrize("mapping", ["thread_per_env", "lanes_per_env", "block_per_env"])
@pytest.mark.parametrize("variant", cases.VARIANTS)
def test_generic_kernels(variant, mapping):
    case = CASES[variant]
    for first, n in case.ranges():
        _check(_run(case, _tables(case, mapping), first, n), case, first, n, f"{mapping} {variant} {first}+{n}")


@pytest.mark.parametrize("variant", cases.VARIANTS)
def test_specialised_and_tile_kernels(variant):
    case = CASES[variant]
    _specialise(case.desc)
    mappings = ["specialized"]
    probe = _tables(case, "specialized")
    assert probe.specialization >= 0
    if _native.load().vmas_b200_specialization_has_tile(probe.specialization):
        mappings.append("tile")
    for mapping in mappings:
        for first, n in case.ranges():
            _check(_run(case, _tables(case, mapping), first, n), case, first, n, f"{mapping} {variant} {first}+{n}")


def _nan_scenario():
    from crafted import _ns

    ns = _ns("vectorizedmultiagentsimulator_b200")

    class NanAction(ns["BaseScenario"]):
        def make_world(self, batch_dim, device, **kwargs):
            world = ns["World"](batch_dim, device, dt=0.1, substeps=2, drag=0.1)
            world.add_agent(ns["Agent"](name="ranged", shape=ns["Sphere"](0.05), collide=False, f_range=0.5,
                                        v_range=0.8, u_range=1.0))
            world.add_agent(ns["Agent"](name="free", shape=ns["Sphere"](0.05), collide=False, u_range=1.0))
            return world

        def reset_world_at(self, env_index=None):
            for a in self.world.agents:
                a.set_pos(torch.zeros(self.world.batch_dim, 2, device=self.world.device), batch_index=env_index)

        def reward(self, agent):
            return torch.zeros(self.world.batch_dim, device=self.world.device)

        def observation(self, agent):
            return agent.state.vel

    return NanAction()


def test_nan_action_stays_nan_through_f_range():
    B = 33
    actions = [torch.full((B, 2), 0.25), torch.full((B, 2), -0.25)]
    actions[0][5, 0] = math.nan
    actions[0][7, 1] = math.nan
    out = {}
    for device in ("cpu", "cuda"):
        if device == "cpu":  # (the oracle env asserts at once unless told not to: its physics is the reference)
            with use_oracle():
                env = b200.make_env(_nan_scenario(), num_envs=B, device=device, seed=0, clamp_actions=False,
                                    action_checks="off")
                env.reset()
                env.step([a.clone() for a in actions])
        else:
            env = b200.make_env(_nan_scenario(), num_envs=B, device=device, seed=0, clamp_actions=False)
            env.reset()
            env.step([a.clone().to(device) for a in actions])
            torch.cuda.synchronize()
            with pytest.raises(AssertionError):
                env.check_actions_now()
        agent = env.agents[0]
        out[device] = (agent.state.force.cpu().clone(), agent.state.vel.cpu().clone(), agent.state.pos.cpu().clone())
    force, vel, pos = out["cuda"]
    assert torch.isnan(force[5, 0]) and torch.isnan(force[7, 1]), "the NaN action must stay NaN through f_range"
    assert torch.isnan(vel[5, 0]) and torch.isnan(vel[7, 1]) and torch.isnan(pos[5, 0])
    for got, want in zip(out["cuda"], out["cpu"]):
        assert torch.equal(torch.isnan(got), torch.isnan(want))
        ok = ~torch.isnan(want)
        assert torch.equal(got[ok], want[ok]) if EXACT else torch.allclose(got[ok], want[ok], rtol=1e-5, atol=1e-6)
