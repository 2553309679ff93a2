"""16-bit observations on the GPU: every way of issuing a step rounds exactly like ``.to(obs_dtype)``.

An env with ``obs_dtype=torch.float16 | torch.bfloat16`` rounds its observations where the step already writes or
copies them: eagerly the hand-out ``.to()``, in a captured step the hand-out copy (converting segments), in the
direct two-launch step the observation gather, in the whole-step kernel its epilogue.  Each must hand out the
eager fp32 env's observations ``.to(obs_dtype)``, bit for bit, and leave everything else bit-identical — without a
launch of its own.  The rounding edges (midpoints, subnormals, fp16 overflow, +-0, inf, NaN) go through the one-kernel
step of a scenario whose observations are its agents' positions, and through the converting copy entry point.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from test_obs_dtype_hostsim import edge_values
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator import observe as O
from vectorizedmultiagentsimulator_b200.simulator.core import Agent, Sphere, World
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E
from vectorizedmultiagentsimulator_b200.simulator.program import StepProgram
from vectorizedmultiagentsimulator_b200.simulator.scenario import BaseScenario

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
DTYPES = [torch.float16, torch.bfloat16]
IDS = ["fp16", "bf16"]

VARIANTS = {
    "one kernel": dict(),
    "whole-step kernel": dict(_INGEST_IN_KERNEL=False),
    "copied results": dict(_WRITE_RESULTS_IN_PLACE=False),
    "two launches": dict(_WHOLE_STEP_KERNEL=False),
    "graph launch": dict(_DIRECT_STEP=False),
    "torch replay": dict(_ONE_CALL_STEP=False),
}


def rounded(got, want32, dtype):
    """``got`` is ``want32.to(dtype)``: bit for bit (NaN where ``want32`` is NaN) in the exact build; in the
    fast-arithmetic build the fp32 values agree to the parity tolerance only, and so do their roundings."""
    if got.dtype != dtype or got.shape != want32.shape:
        return False
    want = want32.to(dtype)
    if not EXACT:
        return same_result(got.float(), want.float(), atol=2e-3, rtol=1e-2)
    nan = want32.isnan()
    return torch.equal(got.isnan(), nan) and torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan])


def check_step(got, want, dtype, what):
    g_obs, w_obs = flatten(got[0]), flatten(want[0])
    assert len(g_obs) == len(w_obs), what
    for i, (g, w) in enumerate(zip(g_obs, w_obs)):
        ok = rounded(g, w, dtype) if w.dtype == torch.float32 else torch.equal(g, w)
        assert ok, f"{what}: observation leaf {i}"
    for i, (g, w) in enumerate(zip(flatten(got[1:]), flatten(want[1:]))):
        assert same_result(g, w, atol=2e-4), f"{what}: result {i}"


def _make(name, kwargs, n_envs, monkeypatch, flags, **env_kw):
    with monkeypatch.context() as m:
        for k, v in flags.items():
            m.setattr(E, k, v)
        # (the whole-step kernels of the 16-bit rows are compiled when the step is captured: wait for them)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)
        env = b200.make_env(name, num_envs=n_envs, device="cuda", seed=0, **env_kw, **kwargs)
        env.reset()
        if env.cuda_graph:  # (the flags are read when the step is captured: warm-up steps + capture happen here)
            for _ in range(4):
                env.step([torch.zeros(n_envs, env.get_agent_action_size(a), device="cuda") for a in env.agents])
    return env


CASES = [
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("navigation", dict(n_agents=4)),
    ("flocking", dict(n_agents=5)),
]


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name,kwargs", CASES, ids=[c[0] for c in CASES])
def test_every_way_of_issuing_a_step_rounds_like_to(name, kwargs, dtype, monkeypatch):
    n = 96
    eager32 = _make(name, kwargs, n, monkeypatch, {})
    envs = {"eager": _make(name, kwargs, n, monkeypatch, {}, obs_dtype=dtype)}
    for label, flags in VARIANTS.items():
        envs[label] = _make(name, kwargs, n, monkeypatch, flags, cuda_graph=True, obs_dtype=dtype)
    for env in envs.values():
        sync_env(eager32, env)
    gen = torch.Generator().manual_seed(5)
    for t in range(10):
        actions = [(torch.rand(n, eager32.get_agent_action_size(a), generator=gen) * 2 - 1).cuda() for a in eager32.agents]
        want = eager32.step([x.clone() for x in actions])
        for label, env in envs.items():
            got = env.step([x.clone() for x in actions])
            check_step(got, want, dtype, f"{name} {label} step {t}")
            for k in ("pos", "vel", "rot", "ang_vel"):
                assert same_result(getattr(env.world.slab, k), getattr(eager32.world.slab, k), atol=2e-4), f"{label} {k}"
            if not EXACT:
                sync_env(eager32, env)
        if t == 5:  # a partial reset in between
            want_obs = eager32.reset_at(7)
            for label, env in envs.items():
                got_obs = env.reset_at(7)
                sync_env(eager32, env)
                for i, (g, w) in enumerate(zip(flatten(got_obs), flatten(want_obs))):
                    assert rounded(g, w, dtype), f"{name} {label} reset_at obs {i}"
    assert all(o.dtype == dtype for o in flatten(got[0]))
    one, whole, copied, two = (envs[k] for k in ("one kernel", "whole-step kernel", "copied results", "two launches"))
    if name == "balance":
        assert one._one_call.c.ingest_in_kernel == 1 and one._one_call.c.fused_kernel > 0 and one._one_call.c.n_segs == 0
        assert whole._one_call.c.n_segs == 0 and whole._one_call.c.obs_block >= 0 and whole._one_call.c.obs_dtype > 0
        assert copied._one_call.c.obs_dtype == 0 and copied._one_call.c.n_segs > 0  # (rounded by the hand-out copy)
        assert two._one_call.direct and two._one_call.c.fused_kernel == 0 and two._one_call.c.obs_dtype > 0
    elif name == "transport":
        assert one._one_call.c.ingest_in_kernel == 1 and one._one_call.c.fused_kernel > 0
    else:  # (LIDAR columns: the captured graph, then the hand-out copy)
        assert one._one_call is None or not one._one_call.direct


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_launch_counts_do_not_change(dtype, monkeypatch):
    """The one-kernel step stays ONE launch with nothing left to copy; copied results stay two (the whole-step
    kernel, then ONE hand-out copy that rounds on the way); the direct two-launch step stays three."""
    n = 96
    counts = {}
    for obs_dtype in (torch.float32, dtype):
        for label in ("one kernel", "copied results", "two launches", "torch replay"):
            env = _make("balance", dict(n_agents=4), n, monkeypatch, VARIANTS[label], cuda_graph=True, obs_dtype=obs_dtype)
            backend = env.world._get_backend()
            before = backend.launches
            env.step([torch.zeros(n, 2, device="cuda") for _ in env.agents])
            counts[(obs_dtype, label)] = backend.launches - before
            if label == "one kernel":
                assert env._one_call.c.n_segs == 0 and env._one_call.c.ingest_in_kernel == 1
    for label in ("one kernel", "copied results", "two launches", "torch replay"):
        assert counts[(dtype, label)] == counts[(torch.float32, label)], label
    assert counts[(dtype, "one kernel")] == 1 and counts[(dtype, "copied results")] == 2


class EdgeScenario(BaseScenario):
    """Four far-apart sphere agents that do not move (no collisions, gravity or semidims; not movable), whose
    positions are set from ``values`` (8 per env); each agent observes all four positions, a blank column and its
    rotation (``odd``: and its angular velocity, an odd width), through a step program and an observation plan."""

    def make_world(self, batch_dim, device, **kwargs):
        self.values = kwargs.pop("values")
        odd = kwargs.pop("odd", False)
        world = World(batch_dim, device)
        for i in range(4):
            world.add_agent(Agent(name=f"agent_{i}", shape=Sphere(0.05), collide=False, movable=False))
        self._plan = O.ObservationPlan(
            [[O.pos(b) for b in world.agents] + [O.blank(1), O.rot(a)] + ([O.ang_vel(a)] if odd else [])
             for a in world.agents]
        )
        self._prog = None
        return world

    def reset_world_at(self, env_index=None):
        vals = self.values.to(self.world.device).reshape(self.world.batch_dim, 4, 2)
        for k, agent in enumerate(self.world.agents):
            agent.set_pos(vals[:, k] if env_index is None else vals[env_index, k], batch_index=env_index)

    def _step_program(self):
        if self._prog is None:
            p = StepProgram(self.world)
            p.out_rew = p.store(p.const(0.0))
            p.out_done = p.store(p.lt(p.const(1.0), p.const(0.0)))
            self._prog = p.finalize()
        return self._prog

    def _observation_plan(self):
        return self._plan

    def reward(self, agent):
        if agent is self.world.agents[0]:
            self._obs_all = self._step_program().run(observe=self._plan)
        return self._prog.out_rew.tensor

    def observation(self, agent):
        if getattr(self, "_obs_all", None) is None:
            self._obs_all = self.world.observe(self._plan)
        row = self._obs_all[self.world.agents.index(agent)]
        if agent is self.world.agents[-1]:
            self._obs_all = None
        return row

    def done(self):
        return self._step_program().out_done.tensor

    def info(self, agent):
        return {}


@pytest.mark.parametrize("odd", [False, True], ids=["width10", "width11"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_one_kernel_step_rounds_the_edges_like_to(dtype, odd, monkeypatch):
    x = torch.from_numpy(edge_values())
    x = torch.cat([x, torch.zeros((-x.numel()) % 8)])
    n = x.numel() // 8
    env = _make(EdgeScenario(), dict(values=x, odd=odd), n, monkeypatch, {}, cuda_graph=True, obs_dtype=dtype)
    assert env._one_call.c.fused_kernel > 0 and env._one_call.c.ingest_in_kernel == 1 and env._one_call.c.n_segs == 0
    pos = x.reshape(n, 4, 2).to("cuda")
    for t in range(2):
        obs = env.step([torch.zeros(n, 2, device="cuda") for _ in env.agents])[0]
        for k, row in enumerate(obs):
            assert row.dtype == dtype
            assert rounded(row[:, :8], pos.reshape(n, 8), dtype), f"step {t} agent {k}: positions"
            assert torch.equal(row[:, 9], torch.zeros(n, dtype=dtype, device="cuda"))  # (rotation)
    assert torch.equal(env.world.slab.pos.reshape(n, 8).view(torch.int32), pos.reshape(n, 8).view(torch.int32)), "moved"


def test_converting_copy_rounds_the_edges_like_to():
    """``vmas_b200_copy_buffers_convert`` on the edge set: heads and tails not 16-byte aligned, destinations not
    8-byte aligned, next to a plain copy segment."""
    lib = _native.load()
    x = torch.from_numpy(edge_values()).cuda()
    n = x.numel()
    kinds = {torch.float16: _native.DTYPE_F16, torch.bfloat16: _native.DTYPE_BF16}
    plain_src = torch.arange(1000, dtype=torch.uint8, device="cuda")
    for dtype, kind in kinds.items():
        for src_off, dst_off in ((0, 0), (1, 0), (3, 1), (0, 3), (2, 2), (5, 7)):
            src = x[src_off:]
            dst = torch.full((n + 16,), float("nan"), dtype=dtype, device="cuda")
            out = dst[dst_off : dst_off + src.numel()]
            plain_dst = torch.zeros(1001, dtype=torch.uint8, device="cuda")
            segs = (_native.CopySegmentC * 2)()
            segs[0].src, segs[0].dst, segs[0].bytes = src.data_ptr(), out.data_ptr(), src.numel() * 4
            segs[1].src, segs[1].dst, segs[1].bytes = plain_src.data_ptr(), plain_dst.data_ptr() + 1, 1000
            k = (C.c_int32 * 2)(kind, _native.DTYPE_F32)
            assert lib.vmas_b200_copy_buffers_convert(segs, k, 2, None) == 1
            torch.cuda.synchronize()
            assert rounded(out, src, dtype), f"{dtype} offsets {src_off}, {dst_off}"
            assert dst[:dst_off].isnan().all() and dst[dst_off + src.numel():].isnan().all(), "wrote outside"
            assert torch.equal(plain_dst[1:], plain_src) and int(plain_dst[0]) == 0
    bad = (C.c_int32 * 1)(_native.DTYPE_F16)
    one = (_native.CopySegmentC * 1)()
    one[0].src, one[0].dst, one[0].bytes = x.data_ptr(), x.data_ptr(), 6  # (not whole fp32 values)
    assert lib.vmas_b200_copy_buffers_convert(one, bad, 1, None) < 0
