"""The host side of the device reset, without a GPU.

``CudaBackend.reset_state`` / ``CudaBackend.spawn`` fill the C-ABI structs (``VmasSpawn``: entity
indices, device pointers, strides, the Philox seed / stream / episode counters).  Here the two
library calls are replaced by a stand-in that *decodes those structs from raw memory* and runs the
numpy oracle on what it finds, so everything above the ABI — ``World.reset``,
``World.spawn_positions``, ``ScenarioUtils``, the scenarios' ``reset_world_at`` with an index or a
mask, ``Environment.reset_at`` — runs exactly as it does on a CUDA world.  (The kernels themselves
are checked against the same oracle on the GPU: ``tests/test_reset_gpu.py``.)
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import reset as R
from oracle.backend import OracleBackend
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.backend import CudaBackend
from vectorizedmultiagentsimulator_b200.simulator.core import World


def _view(ptr, shape, ctype, dtype):
    """numpy view of the host memory a struct field points at."""
    n = int(np.prod(shape))
    return np.ctypeslib.as_array((ctype * n).from_address(ptr)).view(dtype).reshape(shape)


class DecodingNative:
    """Stands in for ``_native.reset_state`` / ``_native.spawn_entities``."""

    MAX_SPAWN = _native.MAX_SPAWN
    SpawnC = _native.SpawnC

    def __init__(self):
        self.calls = []

    class SlabHandle:  # the stand-in needs the slab itself, not its device pointers
        def __init__(self, slab):
            self.slab = slab

    def reset_state(self, lib, handle, env_index, env_mask, reset_count):
        slab = handle.slab
        B = slab.batch_dim
        mask = None if env_mask is None else _view(env_mask.data_ptr(), (B,), C.c_uint8, np.uint8)
        envs = torch.from_numpy(R.selected_envs(B, env_index, mask))
        for t in slab.tensors():
            t[envs] = 0.0
        if reset_count is not None:
            _view(reset_count.data_ptr(), (B,), C.c_int32, np.int32)[envs.numpy()] += 1
        return 1

    def spawn_entities(self, lib, handle, sp):
        slab = handle.slab
        B = slab.batch_dim
        index = None if sp.env_index < 0 else sp.env_index
        mask = _view(sp.env_mask, (B,), C.c_uint8, np.uint8) if sp.env_mask else None
        occupied = None
        if sp.occupied:
            assert sp.occupied_env_stride in (0, sp.n_occupied * 2)
            rows = B if sp.occupied_env_stride else 1
            occupied = _view(sp.occupied, (rows, sp.n_occupied, 2), C.c_float, np.float32).copy()
        pos = slab.pos.contiguous().numpy().copy()
        out, exhausted = R.spawn_entities(
            pos,
            [sp.entity[i] for i in range(sp.n_spawn)],
            min_dist=sp.min_dist,
            x_bounds=(sp.x_lo, sp.x_hi),
            y_bounds=(sp.y_lo, sp.y_hi),
            seed=sp.seed,
            stream_id=sp.stream_id,
            reset_count=_view(sp.reset_count, (B,), C.c_int32, np.int32) if sp.reset_count else None,
            occupied_entities=[sp.occupied_entity[i] for i in range(sp.n_occupied_entities)],
            occupied=occupied,
            env_index=index,
            env_mask=mask,
            max_tries=sp.max_tries,
            env_offset=sp.env_offset,
        )
        slab.pos.copy_(torch.from_numpy(pos))
        if sp.out:
            envs = R.selected_envs(B, index, mask)
            _view(sp.out, (B, sp.n_spawn, 2), C.c_float, np.float32)[envs] = out[envs]
        if sp.status:
            _view(sp.status, (1,), C.c_int32, np.int32)[0] += exhausted
        self.calls.append(dict(n=sp.n_spawn, stream=sp.stream_id, env_index=sp.env_index, seed=sp.seed))
        return 1


class HostPathBackend(OracleBackend):
    """CPU oracle physics + the product's reset marshalling (``CudaBackend.reset_state`` / ``spawn``)."""

    def __init__(self, world):
        super().__init__(world)
        self._native = DecodingNative()
        self.lib = None
        self.device = torch.device("cpu")
        self.launches = 0

    _selection = staticmethod(CudaBackend._selection)
    _slab_handle = CudaBackend._slab_handle
    _slab_index_of = CudaBackend._slab_index_of
    reset_state = CudaBackend.reset_state
    spawn = CudaBackend.spawn


@pytest.fixture
def device_reset_on_cpu(monkeypatch):
    monkeypatch.setattr(World, "_backend_factory", staticmethod(lambda world: HostPathBackend(world)))
    monkeypatch.setattr(World, "uses_device_reset", property(lambda self: True))


def _slab(env):
    return {k: v.clone() for k, v in env.world.slab.state_dict().items()}


CASES = [
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("navigation", dict(n_agents=4)),
    ("flocking", dict(n_agents=5)),
]


@pytest.mark.parametrize("name,kwargs", CASES)
def test_masked_reset_equals_one_reset_at_per_env(device_reset_on_cpu, name, kwargs):
    import vectorizedmultiagentsimulator_b200 as b200

    n = 24
    a = b200.make_env(name, num_envs=n, device="cpu", seed=4, **kwargs)
    b = b200.make_env(name, num_envs=n, device="cpu", seed=4, **kwargs)
    assert all(torch.equal(x, y) for x, y in zip(_slab(a).values(), _slab(b).values()))  # same seed, same layout
    gen = torch.Generator().manual_seed(2)
    for _ in range(2):
        act = [torch.rand(n, 2, generator=gen) * 2 - 1 for _ in a.agents]
        a.step([t.clone() for t in act])
        b.step([t.clone() for t in act])
    before = _slab(a)
    flagged = [0, 5, 6, 23]
    mask = torch.zeros(n, dtype=torch.bool)
    mask[flagged] = True
    obs_a = a.reset_at(mask)
    for i in flagged:
        obs_b = b.reset_at(i)
    after_a, after_b = _slab(a), _slab(b)
    for k in after_a:
        assert torch.equal(after_a[k][~mask], before[k][~mask]), f"{name}: {k} of an unflagged env changed"
        assert torch.equal(after_a[k], after_b[k]), f"{name}: {k}"
    assert all(torch.equal(x, y) for x, y in zip(obs_a, obs_b))
    assert float(after_a["vel"][mask].abs().max()) == 0.0
    for agent in a.world.policy_agents:  # the action buffers are cleared like Agent._reset does
        assert not agent.action.u[mask].any() and agent.action.u[~mask].any()
    assert a.world.reset_count.tolist() == [1 + int(m) for m in mask.tolist()]
    assert a.world.spawn_failures() == 0


def test_spawn_calls_carry_seed_stream_and_selection(device_reset_on_cpu):
    import vectorizedmultiagentsimulator_b200 as b200

    env = b200.make_env("navigation", num_envs=8, device="cpu", seed=21, n_agents=3)
    calls = env.world._get_backend()._native.calls
    # one call for the agents, then one per goal; numbered from 0 within the reset; all envs
    assert [(c["n"], c["stream"], c["env_index"]) for c in calls] == [(3, 0, -1), (1, 1, -1), (1, 2, -1), (1, 3, -1)]
    assert {c["seed"] for c in calls} == {21}
    del calls[:]
    env.reset_at(5)
    assert [(c["stream"], c["env_index"]) for c in calls] == [(0, 5), (1, 5), (2, 5), (3, 5)]
    del calls[:]
    env.seed(99)
    env.reset()
    assert {c["seed"] for c in calls} == {99}
    pts = torch.stack([a.state.pos for a in env.world.agents] + [a.goal.state.pos for a in env.world.agents], dim=1)
    d = torch.cdist(pts, pts) + torch.eye(6) * 10
    assert float(d.min()) >= env.scenario.min_distance_between_entities - 1e-6


def test_long_entity_lists_are_chained(device_reset_on_cpu):
    from vectorizedmultiagentsimulator_b200.simulator.core import Landmark, Sphere
    from vectorizedmultiagentsimulator_b200.simulator.utils import ScenarioUtils

    world = World(4, "cpu")
    ents = [Landmark(name=f"l{i}", shape=Sphere(0.01)) for i in range(70)]
    for e in ents:
        world.add_landmark(e)
    world.reset(None)
    ScenarioUtils.spawn_entities_randomly(ents, world, None, 0.05, (-1, 1), (-1, 1))
    calls = world._get_backend()._native.calls
    assert [c["n"] for c in calls] == [64, 6]
    pts = torch.stack([e.state.pos for e in ents], dim=1)
    d = torch.cdist(pts, pts) + torch.eye(70) * 10
    assert float(d.min()) >= 0.05 - 1e-6  # the second launch kept away from the first one's draws


@pytest.mark.parametrize("name,kwargs", CASES)
@pytest.mark.parametrize("terminated_truncated", [False, True])
def test_auto_reset_equals_step_then_reset_at_dones(device_reset_on_cpu, name, kwargs, terminated_truncated):
    """``auto_reset=True``: the step's rewards / dones, then the observations ``reset_at(dones)`` would
    return.  Episodes end at different times (staggered step counters against ``max_steps``)."""
    import vectorizedmultiagentsimulator_b200 as b200

    n = 12
    opts = dict(num_envs=n, device="cpu", seed=8, max_steps=4, terminated_truncated=terminated_truncated, **kwargs)
    auto = b200.make_env(name, auto_reset=True, **opts)
    manual = b200.make_env(name, **opts)
    stagger = torch.arange(n, dtype=torch.float32) % 4
    auto.steps.copy_(stagger)
    manual.steps.copy_(stagger)
    gen = torch.Generator().manual_seed(1)
    finished_total = 0
    for t in range(9):
        act = [torch.rand(n, 2, generator=gen) * 2 - 1 for _ in auto.agents]
        got = auto.step([a.clone() for a in act])
        want = manual.step([a.clone() for a in act])
        finished = (want[2] | want[3]) if terminated_truncated else want[2]
        finished_total += int(finished.sum())
        want_obs = manual.reset_at(finished)
        for g, w in zip(got[0], want_obs):
            assert torch.equal(g, w), f"{name} step {t}: observations"
        for g, w in zip(got[1], want[1]):
            assert torch.equal(g, w), f"{name} step {t}: rewards"
        for k in range(2, 4 if terminated_truncated else 3):
            assert torch.equal(got[k], want[k]), f"{name} step {t}: dones"
        assert torch.equal(auto.steps, manual.steps)
        for x, y in zip(_slab(auto).values(), _slab(manual).values()):
            assert torch.equal(x, y)
    assert finished_total >= 2 * n  # every env ended at least two episodes
    assert auto.world.reset_count.min() >= 3


def test_auto_reset_needs_a_mask_capable_scenario():
    import vectorizedmultiagentsimulator_b200 as b200
    from oracle.backend import use_oracle
    from vectorizedmultiagentsimulator_b200.scenarios import balance

    class IndexOnly(balance.Scenario):
        supports_masked_reset = False

    with use_oracle():
        with pytest.raises(NotImplementedError):
            b200.make_env(IndexOnly(), num_envs=4, device="cpu", seed=0, n_agents=3, auto_reset=True)


@pytest.mark.parametrize("name,kwargs", CASES)
def test_shards_reset_like_the_unsharded_job(device_reset_on_cpu, name, kwargs):
    """``shard.make_shard_env``: a shard's layouts (initial and after a masked reset) are the matching
    slice of the unsharded job's — what makes results independent of the number of GPUs."""
    import vectorizedmultiagentsimulator_b200 as b200
    from vectorizedmultiagentsimulator_b200 import shard

    total = 22
    full = shard.make_shard_env(name, total, 0, 1, "cpu", seed=6, **kwargs)
    plain = b200.make_env(name, num_envs=total, device="cpu", seed=6, **kwargs)
    assert torch.equal(full.world.slab.pos, plain.world.slab.pos)  # a job of one shard == a plain env
    mask = torch.rand(total, generator=torch.Generator().manual_seed(0)) < 0.4
    full.reset_at(mask)
    for rank in range(3):
        lo, hi = shard.shard_bounds(total, rank, 3)
        part = shard.make_shard_env(name, total, rank, 3, "cpu", seed=6, **kwargs)
        assert part.num_envs == hi - lo and part.world.env_offset == lo
        part.reset_at(mask[lo:hi])
        for (k, got), want in zip(_slab(part).items(), _slab(full).values()):
            assert torch.equal(got, want[lo:hi]), f"{name} rank {rank}: {k}"

